/* Streamed input from plain C: the rows of a seeded table are pushed in uneven blocks from two alternating pinned
 * buffers, round after round while the engine asks for them again, the way a host decodes ClickHouse blocks while the
 * previous one is on the bus.  The same table is then run once through tad_submit for comparison.
 *
 *   gcc -std=c99 -Wall -Iinclude examples/tad_stream.c -Ltheia_b200 -ltheia_tad -Wl,-rpath,$PWD/theia_b200 -o tad_stream
 *   ./tad_stream [budget_bytes]     # needs a H100; a budget (>= 64 MiB) makes the job run in several rounds
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "theia_tad.h"

enum { SERIES = 2000, POINTS = 150, ROWS = SERIES * POINTS, BLOCK_CAP = 5000 };

/* row i of the table: a function of i alone, so every round can produce it again without holding the table */
static void make_row(uint64_t i, tad_columns *c, uint64_t at)
{
    const uint32_t s = (uint32_t)(i % SERIES), p = (uint32_t)(i / SERIES);
    uint32_t x = (uint32_t)i * 2654435761u ^ 0x9e3779b9u;
    x ^= x >> 15; x *= 2246822519u; x ^= x >> 13;
    c->src_ip[at] = 0x0A000000u | (s * 7919u & 0xFFFFFFu);
    c->dst_ip[at] = 0x0A800000u | (s * 104729u & 0x7FFFFFu);
    c->src_port[at] = (uint16_t)(1024 + s % 50000);
    c->dst_port[at] = 5201;
    c->proto[at] = 6;
    c->flow_start[at] = 1660199214u;
    c->flow_end[at] = 1660202814u + 60u * p;
    c->value[at] = 4000000000ull + x % 1000000u + (x % 97 == 0 ? 40000000000ull : 0);
}

static int wait_job(tad_job *job, tad_status *st, const char *what)
{
    tad_wait(job, -1, st);
    if (st->state != TAD_STATE_COMPLETED) {
        fprintf(stderr, "%s failed: %s\n", what, st->err_msg);
        return 1;
    }
    return 0;
}

int main(int argc, char **argv)
{
    tad_config cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.world_size = 1;
    tad_ctx *ctx = NULL;
    int rc = tad_init(&cfg, &ctx);
    if (rc != TAD_OK) {
        fprintf(stderr, "tad_init: %s\n", tad_strerror(rc));
        return 1;
    }
    if (argc > 1 && (rc = tad_set_memory_budget(ctx, strtoull(argv[1], NULL, 10))) != TAD_OK) {
        fprintf(stderr, "tad_set_memory_budget: %s\n", tad_strerror(rc));
        return 1;
    }
    tad_job_spec spec;
    memset(&spec, 0, sizeof(spec));
    spec.algo = TAD_ALGO_EWMA;
    spec.reducer = TAD_REDUCE_MAX;
    strncpy(spec.id, "5ca1ab1e-0000-4000-8000-000000000002", sizeof(spec.id) - 1);

    /* two pinned blocks: block k+1 is filled while block k is copied */
    tad_columns buf[2];
    if (tad_alloc_columns(ctx, BLOCK_CAP, TAD_MEM_HOST, &buf[0]) != TAD_OK ||
        tad_alloc_columns(ctx, BLOCK_CAP, TAD_MEM_HOST, &buf[1]) != TAD_OK)
        return 1;
    tad_job *job = NULL;
    rc = tad_submit_stream(ctx, &spec, ROWS, &job);
    int rounds = 0;
    int32_t again = 1;
    while (rc == TAD_OK && again) {
        uint64_t next = 0;
        int k = 0;
        for (uint64_t i = 0; rc == TAD_OK && i < ROWS; k++) {
            uint64_t n = 1 + (next = next * 6364136223846793005ull + 1442695040888963407ull + (uint64_t)rounds) % BLOCK_CAP;
            if (n > ROWS - i) n = ROWS - i;                /* uneven block sizes, 1 .. BLOCK_CAP rows */
            tad_columns *b = &buf[k & 1];
            for (uint64_t j = 0; j < n; j++) make_row(i + j, b, j);
            b->rows = n;
            rc = tad_stream_push(job, b);
            i += n;
        }
        if (rc == TAD_OK) rc = tad_stream_end(job, &again);
        rounds++;
    }
    tad_status st;
    if (rc != TAD_OK) {
        tad_poll(job, &st);
        fprintf(stderr, "streamed job: %s: %s\n", tad_strerror(rc), st.err_msg);
        return 1;
    }
    if (wait_job(job, &st, "streamed job")) return 1;
    uint32_t passes = 0;
    tad_job_memory(job, &passes, NULL);
    tad_rows rows;
    tad_result(job, &rows);
    const unsigned long long streamed = (unsigned long long)rows.rows;
    printf("streamed: %llu rows in, %llu series, %llu anomalous rows, %d rounds, %u passes\n",
           (unsigned long long)st.rows_in, (unsigned long long)st.series, streamed, rounds, passes);
    tad_release(job);
    tad_free_columns(ctx, &buf[0]);
    tad_free_columns(ctx, &buf[1]);

    /* the same table in one tad_submit */
    tad_columns cols;
    if (tad_alloc_columns(ctx, ROWS, TAD_MEM_HOST, &cols) != TAD_OK) return 1;
    for (uint64_t i = 0; i < ROWS; i++) make_row(i, &cols, i);
    cols.rows = ROWS;
    if (tad_submit(ctx, &spec, &cols, &job) != TAD_OK || wait_job(job, &st, "one-shot job")) return 1;
    tad_result(job, &rows);
    printf("one-shot: %llu anomalous rows\n", (unsigned long long)rows.rows);
    printf("%s\n", (unsigned long long)rows.rows == streamed ? "same result count" : "result counts differ");
    tad_release(job);
    tad_free_columns(ctx, &cols);
    tad_shutdown(ctx);
    return (unsigned long long)rows.rows == streamed ? 0 : 1;
}
