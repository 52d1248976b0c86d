/* c_abi_demo.c -- the C ABI (include/summerset_b200.h) used from plain C, the way a Rust `extern "C"` shim
 * would drive it: no torch, no C++ -- pointers and sizes only.
 *
 * One tick of a batched RSPaxos leader for G groups:
 *   host payloads -> device arena                         (ss_copy_h2d)
 *   RS(3,2)-encode every group's request batch + tally the acks that arrived   (ss_accept_step_fused_dev)
 *   commit_bar[] back to the host                         (ss_copy_d2h)
 * then a follower-side reconstruct of a codeword that lost two shards (ss_rs_reconstruct, host slices),
 * then the batched engine (ss_engine_*): propose slot 0 for every group, feed AcceptReply records, tick until the
 * instances commit -- what the Rust shim's run() loop does once per event-loop turn.
 *
 * build: gcc -O2 examples/c_abi_demo.c -Iinclude -Lsummerset_b200 -lsummerset_b200 -Wl,-rpath,$PWD/summerset_b200 -o c_abi_demo
 * Without an sm_90 GPU it prints the library's refusal (there is no CPU fallback) and exits 3.
 */
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "summerset_b200.h"

#define CHECK(call)                                                                  \
    do {                                                                             \
        int rc_ = (call);                                                            \
        if (rc_ != SS_OK) {                                                          \
            fprintf(stderr, "%s -> %d: %s\n", #call, rc_, ss_last_error());          \
            return rc_ == SS_ERR_NO_DEVICE ? 3 : 1;                                  \
        }                                                                            \
    } while (0)

int main(void) {
    enum { G = 4096, LEN = 4096, D = 3, P = 2, R = 5 };
    const uint32_t L = (LEN + D - 1) / D, DS = (L + 15) / 16 * 16;     /* shard length 1366, padded slot 1376 */
    ss_ctx *ctx = NULL;
    ss_rs_coder *rs = NULL;
    CHECK(ss_ctx_create(0, &ctx));
    CHECK(ss_rs_coder_create(ctx, D, P, &rs));

    /* host side: pinned payloads and ack planes (leader always acks, followers ack 7 of 8 slots) */
    uint8_t *h_data = NULL; uint64_t *h_planes = NULL; uint32_t *h_bar = NULL;
    CHECK(ss_host_alloc(ctx, (size_t)G * LEN, (void **)&h_data));
    CHECK(ss_host_alloc(ctx, (size_t)R * G * 8, (void **)&h_planes));
    CHECK(ss_host_alloc(ctx, (size_t)G * 4, (void **)&h_bar));
    for (size_t i = 0; i < (size_t)G * LEN; ++i) h_data[i] = (uint8_t)(i * 2654435761u >> 13);
    for (int r = 0; r < R; ++r)
        for (int g = 0; g < G; ++g) h_planes[(size_t)r * G + g] = r == 0 ? ~0ull : ~(0x0101010101010101ull << ((g + r) & 7));

    /* device side */
    uint8_t *d_data = NULL, *d_parity = NULL; uint64_t *d_planes = NULL, *d_committed = NULL; uint32_t *d_bar = NULL;
    CHECK(ss_dev_alloc(ctx, (size_t)G * LEN, (void **)&d_data));
    CHECK(ss_dev_alloc(ctx, (size_t)P * G * DS, (void **)&d_parity));
    CHECK(ss_dev_alloc(ctx, (size_t)R * G * 8, (void **)&d_planes));
    CHECK(ss_dev_alloc(ctx, (size_t)G * 8, (void **)&d_committed));
    CHECK(ss_dev_alloc(ctx, (size_t)G * 4, (void **)&d_bar));
    CHECK(ss_copy_h2d(ctx, d_data, h_data, (size_t)G * LEN));
    CHECK(ss_copy_h2d(ctx, d_planes, h_planes, (size_t)R * G * 8));
    /* threshold = majority + fault_tolerance = 3 + 1 (rspaxos/messages.rs:438-440) */
    CHECK(ss_accept_step_fused_dev(rs, d_data, LEN, LEN, G, d_parity, (uint64_t)G * DS, DS, SS_RS_OUT_PADDED16, d_planes, R, 4,
                                   d_committed, d_bar));
    CHECK(ss_copy_d2h(ctx, h_bar, d_bar, (size_t)G * 4));
    CHECK(ss_ctx_sync(ctx));
    unsigned long long slots = 0;
    for (int g = 0; g < G; ++g) slots += h_bar[g];
    printf("fused accept step: %d groups, %llu slots in committed prefixes, kernels launched: %llu\n", G, slots,
           (unsigned long long)ss_ctx_launch_count(ctx));

    /* follower side, one codeword through the crate-shaped calls: encode, lose shards 0 and 3, reconstruct */
    uint8_t shard[D + P][1366], keep0[1366];
    uint8_t *ptr[D + P];
    uint8_t present[D + P] = {1, 1, 1, 1, 1};
    for (int j = 0; j < D + P; ++j) ptr[j] = shard[j];
    memset(shard, 0, sizeof(shard));
    memcpy(shard[0], h_data, L); memcpy(shard[1], h_data + L, L); memcpy(shard[2], h_data + 2 * L, LEN - 2 * L);
    CHECK(ss_rs_encode(rs, ptr, D + P, L));
    int ok = 0;
    CHECK(ss_rs_verify(rs, (const uint8_t *const *)ptr, D + P, L, &ok));
    memcpy(keep0, shard[0], L);
    memset(shard[0], 0xEE, L); memset(shard[3], 0xEE, L);
    present[0] = present[3] = 0;
    CHECK(ss_rs_reconstruct(rs, ptr, present, D + P, L));
    printf("verify after encode: %s; reconstruct of shards {0,3}: %s\n", ok ? "ok" : "MISMATCH",
           memcmp(keep0, shard[0], L) == 0 && present[0] && present[3] ? "bit-exact" : "MISMATCH");
    /* too few shards: refused, nothing written */
    present[0] = present[1] = present[4] = 0;
    int rc = ss_rs_reconstruct(rs, ptr, present, D + P, L);
    printf("3 of 5 missing -> %d (%s)\n", rc, ss_strerror(rc));

    /* ---- the engine: RSPaxos leader state of G groups, n = 5, f = 1 (commit at 4 acks) ---- */
    int eng_ok = 0;
    {
        ss_engine *eng = NULL;
        ss_engine_config cfg;
        memset(&cfg, 0, sizeof cfg);
        cfg.protocol = SS_PROTO_RSPAXOS; cfg.population = R; cfg.fault_tolerance = 1; cfg.data_len = LEN; cfg.keep_slots = 1;
        CHECK(ss_engine_create(ctx, &cfg, G, &eng));
        uint64_t *h_bal = NULL; uint32_t *h_rg = NULL; uint8_t *h_rs = NULL, *h_rp = NULL; uint64_t *h_rb = NULL;
        const size_t NREC = (size_t)G * 4;                   /* replicas 0..3 ack slot 0 of every group */
        CHECK(ss_host_alloc(ctx, (size_t)G * 8, (void **)&h_bal));
        CHECK(ss_host_alloc(ctx, NREC * 4, (void **)&h_rg)); CHECK(ss_host_alloc(ctx, NREC, (void **)&h_rs));
        CHECK(ss_host_alloc(ctx, NREC, (void **)&h_rp)); CHECK(ss_host_alloc(ctx, NREC * 8, (void **)&h_rb));
        for (int g = 0; g < G; ++g) h_bal[g] = 100 + (uint64_t)g;
        for (size_t i = 0; i < NREC; ++i) {
            h_rg[i] = (uint32_t)(i / 4); h_rs[i] = 0; h_rp[i] = (uint8_t)(i % 4);
            h_rb[i] = h_bal[i / 4] + ((i % 64) == 7 ? 1 : 0);                    /* a few stale-ballot replies */
        }
        uint64_t *d_bal = NULL, *d_rb = NULL, *d_newly = NULL; uint32_t *d_rg = NULL; uint8_t *d_rs = NULL, *d_rp = NULL, *planes0 = NULL;
        CHECK(ss_dev_alloc(ctx, (size_t)G * 8, (void **)&d_bal)); CHECK(ss_dev_alloc(ctx, (size_t)G * 8, (void **)&d_newly));
        CHECK(ss_dev_alloc(ctx, NREC * 4, (void **)&d_rg)); CHECK(ss_dev_alloc(ctx, NREC, (void **)&d_rs));
        CHECK(ss_dev_alloc(ctx, NREC, (void **)&d_rp)); CHECK(ss_dev_alloc(ctx, NREC * 8, (void **)&d_rb));
        CHECK(ss_copy_h2d(ctx, d_bal, h_bal, (size_t)G * 8));
        CHECK(ss_copy_h2d(ctx, d_rg, h_rg, NREC * 4)); CHECK(ss_copy_h2d(ctx, d_rs, h_rs, NREC));
        CHECK(ss_copy_h2d(ctx, d_rp, h_rp, NREC)); CHECK(ss_copy_h2d(ctx, d_rb, h_rb, NREC * 8));
        CHECK(ss_engine_set_prepared_ballots(eng, d_bal));
        CHECK(ss_engine_propose(eng, 0, d_data, LEN, NULL, &planes0));          /* shard planes = per-peer send buffers */
        CHECK(ss_engine_ingest(eng, d_rg, d_rs, d_rp, d_rb, NREC));
        CHECK(ss_engine_tick(eng, d_newly));
        ss_engine_view v;
        CHECK(ss_engine_view_get(eng, &v));
        CHECK(ss_copy_d2h(ctx, h_bar, v.commit_bar, (size_t)G * 4));
        CHECK(ss_ctx_sync(ctx));
        unsigned long long committed_groups = 0, stale_groups = 0;
        for (int g = 0; g < G; ++g) committed_groups += h_bar[g] == 1;
        for (size_t i = 0; i < NREC; ++i) stale_groups += (i % 64) == 7;         /* each stale reply leaves its group at 3 acks */
        printf("engine: %llu of %d groups committed slot 0 after 4 acks (%llu groups saw a stale-ballot reply), "
               "threshold %u, shard planes at %p\n", committed_groups, G, stale_groups, v.threshold, (void *)planes0);
        eng_ok = committed_groups + stale_groups == (unsigned long long)G && v.threshold == 4 && planes0 != NULL;
        ss_dev_free(ctx, d_bal); ss_dev_free(ctx, d_newly); ss_dev_free(ctx, d_rg); ss_dev_free(ctx, d_rs); ss_dev_free(ctx, d_rp);
        ss_dev_free(ctx, d_rb);
        ss_host_free(ctx, h_bal); ss_host_free(ctx, h_rg); ss_host_free(ctx, h_rs); ss_host_free(ctx, h_rp); ss_host_free(ctx, h_rb);
        CHECK(ss_engine_destroy(eng));
    }

    ss_dev_free(ctx, d_data); ss_dev_free(ctx, d_parity); ss_dev_free(ctx, d_planes); ss_dev_free(ctx, d_committed); ss_dev_free(ctx, d_bar);
    ss_host_free(ctx, h_data); ss_host_free(ctx, h_planes); ss_host_free(ctx, h_bar);
    ss_rs_coder_destroy(rs);
    ss_ctx_destroy(ctx);
    return (ok && eng_ok && rc == SS_ERR_TOO_FEW_SHARDS_PRESENT) ? 0 : 1;
}
