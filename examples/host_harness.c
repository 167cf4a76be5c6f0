/* A compiled host that drives libb200prover.so through its C ABI only — the role the Rust shim
 * (INTEGRATION.md) plays behind `SingleProverCircuit::prove_with_link_hint`
 * (crates/circuits/circuit-types/src/traits.rs:972-998): load the SRS points, preprocess a circuit,
 * prove, write the proof.  No Python, no torch: plain pointers and sizes.
 *
 * Job file (little-endian), written by tests/test_gpu_harness.py:
 *   u64 log_n, u64 num_inputs, u64 n_srs,
 *   k[5][4], selectors[13][n][4], perm[5n], wires[5][n][4], pub_inputs[num_inputs][4], blinders[17][4],
 *   srs[n_srs][8]                                     (all u64)
 * Output file: b200_proof (1152 bytes) || link polynomial ((n+2) x 4 u64) || 18 VK commitments.
 * Optional bundle file: the two proofs (2 x 1152 bytes) || the link proof (128 bytes) of the witness bundle below.
 *
 *   gcc -O2 -Iinclude examples/host_harness.c -Lrenegade_b200 -lb200prover -Wl,-rpath,'$ORIGIN/../renegade_b200' -o examples/host_harness
 */
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "b200prover.h"

#define CHECK(call)                                                                  \
    do {                                                                             \
        int rc_ = (call);                                                            \
        if (rc_ != B200_OK) {                                                        \
            fprintf(stderr, "%s failed: %d (%s)\n", #call, rc_, b200_last_error()); \
            return 2;                                                                \
        }                                                                            \
    } while (0)

static uint64_t* read_u64s(FILE* f, size_t count) {
    uint64_t* p = (uint64_t*)malloc(count * 8 + 8);
    if (!p || fread(p, 8, count, f) != count) {
        fprintf(stderr, "short job file\n");
        exit(3);
    }
    return p;
}

int main(int argc, char** argv) {
    if (argc != 3 && argc != 4) {
        fprintf(stderr, "usage: %s job.bin proof.bin [bundle.bin]\n", argv[0]);
        return 1;
    }
    FILE* f = fopen(argv[1], "rb");
    if (!f) { perror("job"); return 1; }
    uint64_t hdr[3];
    if (fread(hdr, 8, 3, f) != 3) return 3;
    const unsigned log_n = (unsigned)hdr[0];
    const size_t num_inputs = (size_t)hdr[1], n_srs = (size_t)hdr[2], n = (size_t)1 << log_n;
    uint64_t* k = read_u64s(f, 5 * 4);
    uint64_t* selectors = read_u64s(f, 13 * n * 4);
    uint64_t* perm = read_u64s(f, 5 * n);
    uint64_t* wires = read_u64s(f, 5 * n * 4);
    uint64_t* pub_inputs = read_u64s(f, num_inputs * 4);
    uint64_t* blinders = read_u64s(f, 17 * 4);
    uint64_t* srs = read_u64s(f, n_srs * 8);
    fclose(f);

    b200_ctx* ctx = NULL;
    b200_bases* bases = NULL;
    b200_pk* pk = NULL;
    CHECK(b200_init(0, &ctx));
    fprintf(stderr, "%s\n", b200_version());
    CHECK(b200_bases_load(ctx, (const uint8_t*)srs, n_srs, 0, /*check_on_curve=*/1, &bases));
    CHECK(b200_plonk_preprocess(ctx, bases, log_n, num_inputs, selectors, perm, k, &pk));
    uint64_t vk[18 * 8];
    CHECK(b200_pk_verifying_key(pk, vk, vk + 13 * 8));

    b200_proof proof;
    uint64_t* link = (uint64_t*)calloc((n + 2) * 4, 8);
    CHECK(b200_plonk_prove(ctx, pk, wires, pub_inputs, blinders, &proof, link, NULL));

    /* an unsatisfying witness must come back as an error code, never an abort (SURVEY.md §5.3) */
    wires[4 * (4 * n + num_inputs + 1)] ^= 1u;
    b200_proof bad;
    int rc = b200_plonk_prove(ctx, pk, wires, pub_inputs, blinders, &bad, NULL, NULL);
    if (rc != B200_ERR_UNSATISFIED) {
        fprintf(stderr, "expected B200_ERR_UNSATISFIED, got %d\n", rc);
        return 4;
    }

    /* the same proof through the prover pool (the NativeProofManager-shaped entry point): four jobs on
     * two workers share the key; every result must equal the single-context proof byte for byte */
    wires[4 * (4 * n + num_inputs + 1)] ^= 1u; /* restore the good witness */
    b200_pool* pool = NULL;
    CHECK(b200_pool_create(0, 2, &pool));
    b200_proof pooled[4];
    uint64_t tickets[4];
    for (int i = 0; i < 4; ++i)
        CHECK(b200_pool_submit_prove(pool, pk, wires, pub_inputs, num_inputs, blinders, &pooled[i], NULL, &tickets[i]));
    for (int i = 3; i >= 0; --i) CHECK(b200_pool_wait(pool, tickets[i]));
    for (int i = 0; i < 4; ++i)
        if (memcmp(&pooled[i], &proof, sizeof(proof)) != 0) {
            fprintf(stderr, "pool proof %d differs from the direct proof\n", i);
            return 5;
        }

    /* The same circuit handed over as a host like the reference's holds it: the wiring (the variable on every wire
     * position) and the witness vector.  Here they are recovered from the job's tables: one variable per cycle of the
     * copy permutation.  A key made from the wiring proves from the witness vector alone; proof and public inputs must
     * equal those of b200_plonk_prove on the 5 x n table under the same key, directly, as a batch and through the pool. */
    unsigned* wire_vars = (unsigned*)malloc(5 * n * sizeof(unsigned));
    uint64_t* witness = (uint64_t*)malloc(5 * n * 32);
    size_t num_vars = 0;
    memset(wire_vars, 0xFF, 5 * n * sizeof(unsigned));
    for (size_t p = 0; p < 5 * n; ++p) {
        if (wire_vars[p] != 0xFFFFFFFFu) continue;
        memcpy(witness + 4 * num_vars, wires + 4 * p, 32);
        for (size_t q = p; wire_vars[q] == 0xFFFFFFFFu; q = (size_t)perm[q]) wire_vars[q] = (unsigned)num_vars;
        ++num_vars;
    }
    b200_pk* wpk = NULL;
    CHECK(b200_plonk_preprocess_wiring(ctx, bases, log_n, num_inputs, selectors, wire_vars, num_vars, k, &wpk));
    if (b200_pk_num_vars(wpk) != num_vars || b200_pk_num_vars(pk) != 0) {
        fprintf(stderr, "b200_pk_num_vars: wrong answer\n");
        return 6;
    }
    b200_proof from_table, from_witness[4];
    uint64_t* pub_out = (uint64_t*)calloc(4 * (num_inputs + 1) * 4, 8);
    CHECK(b200_plonk_prove(ctx, wpk, wires, pub_inputs, blinders, &from_table, NULL, NULL));
    CHECK(b200_plonk_prove_witness(ctx, wpk, witness, blinders, &from_witness[0], NULL, NULL, pub_out));
    b200_witness_item items[2] = {{witness, blinders, &from_witness[1], NULL, NULL, pub_out + 4 * num_inputs},
                                  {witness, blinders, &from_witness[2], NULL, NULL, pub_out + 8 * num_inputs}};
    int statuses[2];
    CHECK(b200_plonk_prove_witness_batch(ctx, wpk, items, 2, statuses));
    CHECK(b200_pool_submit_prove_witness(pool, wpk, witness, blinders, &from_witness[3], NULL, pub_out + 12 * num_inputs, &tickets[0]));
    CHECK(b200_pool_wait(pool, tickets[0]));
    for (int i = 0; i < 4; ++i)
        if (memcmp(&from_witness[i], &from_table, sizeof(proof)) != 0 ||
            memcmp(pub_out + 4 * num_inputs * i, pub_inputs, 32 * num_inputs) != 0) {
            fprintf(stderr, "witness proof %d differs from the proof on the expanded table\n", i);
            return 6;
        }

    /* A bundle of witness vectors through the pool, the shape a relayer settles: two proofs of the key from the wiring
     * (the second with its 17 blinders in reverse order) and one link proof between them on rows num_inputs ..
     * num_inputs + 3, where both carry the same witness values.  Each proof must equal the direct one. */
    uint64_t* blinders_rev = (uint64_t*)malloc(17 * 32);
    for (int i = 0; i < 17; ++i) memcpy(blinders_rev + 4 * i, blinders + 4 * (16 - i), 32);
    uint64_t* bundle_polys = (uint64_t*)calloc(2 * (n + 2) * 4, 8);
    b200_proof bundled[2], direct_rev;
    b200_link_proof bundled_link;
    const b200_bundle_witness bw[2] = {{wpk, witness, blinders, &bundled[0], bundle_polys, NULL},
                                       {wpk, witness, blinders_rev, &bundled[1], bundle_polys + (n + 2) * 4, NULL}};
    const b200_bundle_link blink = {0, 1, log_n, num_inputs, 4, &bundled_link};
    CHECK(b200_pool_submit_bundle_witness(pool, bases, bw, 2, &blink, 1, &tickets[0]));
    CHECK(b200_pool_wait(pool, tickets[0]));
    CHECK(b200_plonk_prove_witness(ctx, wpk, witness, blinders_rev, &direct_rev, NULL, NULL, NULL));
    if (memcmp(&bundled[0], &from_table, sizeof(proof)) != 0 || memcmp(&bundled[1], &direct_rev, sizeof(proof)) != 0) {
        fprintf(stderr, "witness bundle proof differs from the direct proof\n");
        return 7;
    }
    if (argc == 4) { /* the bundle's two proofs and its link proof, for the caller to check against the oracle */
        FILE* ob = fopen(argv[3], "wb");
        if (!ob) { perror("bundle out"); return 1; }
        fwrite(bundled, sizeof(b200_proof), 2, ob);
        fwrite(&bundled_link, sizeof(bundled_link), 1, ob);
        fclose(ob);
    }
    b200_pk_free(ctx, wpk);
    b200_pool_destroy(pool);

    FILE* o = fopen(argv[2], "wb");
    if (!o) { perror("out"); return 1; }
    fwrite(&proof, sizeof(proof), 1, o);
    fwrite(link, 8, (n + 2) * 4, o);
    fwrite(vk, 8, 18 * 8, o);
    fclose(o);

    b200_pk_free(ctx, pk);
    b200_bases_free(ctx, bases);
    b200_shutdown(ctx);
    fprintf(stderr, "proof written (%zu bytes)\n", sizeof(proof));
    return 0;
}
