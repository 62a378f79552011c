/*
 * theia_tad.h -- C ABI of the H100-native throughput-anomaly-detection (TAD) engine.
 *
 * This is the drop-in boundary for ONE path of antrea-io/theia: the job that
 * pkg/controller/anomalydetector/controller.go launches as a SparkApplication
 * (startSparkApplication, controller.go:525-698) and that
 * plugins/anomaly-detection/anomaly_detection.py executes.  The reference has no FFI for
 * this path (its boundary is "create a SparkApplication CR, poll it, read ClickHouse"),
 * so every entry point below cites the reference function it replaces; INTEGRATION.md
 * shows the cgo binding a maintainer adds behind the controller's function-variable seam
 * (controller.go:54-59).
 *
 * Conventions: plain C, no callbacks into the host language, no exceptions across the
 * boundary; every function returns 0 (TAD_OK) or a negative tad_error; strings are
 * NUL-terminated UTF-8.  A tad_ctx may be used from several threads (the controller
 * runs 4 workers, pkg/controller/util.go:43); a tad_job belongs to the thread that polls
 * it.  All pinned-host and device memory is owned by the library (Go's GC may move Go
 * memory, so the host shim fills library-owned buffers obtained from tad_alloc_columns).
 */
#ifndef THEIA_TAD_H
#define THEIA_TAD_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TAD_ABI_VERSION 2   /* 2: tad_job_spec.global_rows, TAD_PHASE_SYNC */

typedef enum {
    TAD_OK = 0,
    TAD_ERR_INVALID_ARG = -1,  /* controller.go:527-622 "invalid request: ..." class      */
    TAD_ERR_CUDA = -2,
    TAD_ERR_NOMEM = -3,
    TAD_ERR_NCCL = -4,
    TAD_ERR_STATE = -5,        /* call not legal in the job's current state                */
    TAD_ERR_CANCELLED = -6,
    TAD_ERR_UNSUPPORTED = -7,
    TAD_ERR_INTERNAL = -8
} tad_error;

/* anomaly_detection.py:811 valid_algos; controller.go:527 */
typedef enum { TAD_ALGO_EWMA = 0, TAD_ALGO_ARIMA = 1, TAD_ALGO_DBSCAN = 2 } tad_algo;

/* Stage-A reducer over duplicates of (key, flowEndSeconds): max(throughput) for the
 * per-connection query (anomaly_detection.py:52-61), sum(throughput) for the pod /
 * external / svc aggregated-flow queries (:63-106). */
typedef enum { TAD_REDUCE_MAX = 0, TAD_REDUCE_SUM = 1 } tad_reducer;

/* Job states = ThroughputAnomalyDetectorStatus.State, pkg/apis/crd/v1alpha1/types.go:33-37 */
typedef enum {
    TAD_STATE_NEW = 0, TAD_STATE_SCHEDULED = 1, TAD_STATE_RUNNING = 2,
    TAD_STATE_COMPLETED = 3, TAD_STATE_FAILED = 4
} tad_state;

typedef enum { TAD_MEM_HOST = 0, TAD_MEM_DEVICE = 1 } tad_mem;

/* tad_job_spec.flags */
#define TAD_FLAG_EMIT_ALL 1u   /* emit every point with its flag (parity/debug), not only anomalies */
#define TAD_FLAG_PROFILE  2u   /* record per-phase CUDA-event times into tad_status.phase_ms         */
#define TAD_FLAG_SHARE    4u   /* a streamed job takes part in fit sharing (tad_set_fit_sharing)     */
#define TAD_FLAG_FIT_BESIDE 8u /* an ARIMA job may fit beside another job's fit while fit sharing is  */
                               /* on (tad_set_fit_sharing): a tad_submit job, or a streamed one that  */
                               /* has TAD_FLAG_SHARE too; ignored on EWMA and DBSCAN jobs, on         */
                               /* streamed jobs without TAD_FLAG_SHARE and while sharing is off       */
#define TAD_FLAG_LEND    16u   /* a streamed job lends the GPU to queued EWMA and DBSCAN tad_submit   */
                               /* jobs while it waits for its caller's next block, while fit sharing  */
                               /* is on (tad_set_fit_sharing); ignored on tad_submit jobs and while   */
                               /* sharing is off                                                      */
#define TAD_FLAG_RANK_STREAM 32u /* world_size > 1: a tad_submit_stream job that is this rank's part of a  */
                                 /* job streamed to every rank (see "Several GPUs" under Streamed input); */
                                 /* ignored on one GPU                                                    */

typedef struct tad_ctx tad_ctx;
typedef struct tad_job tad_job;

typedef struct {
    int32_t device;            /* CUDA device ordinal of this process/rank                          */
    int32_t world_size;        /* 1 = single GPU; N = this process is one of N ranks on one host    */
    int32_t rank;
    uint32_t flags;            /* reserved, 0                                                       */
    const void *nccl_unique_id;/* world_size > 1: the 128-byte ncclUniqueId shared by all ranks      */
    size_t nccl_unique_id_bytes;
} tad_config;

/*
 * Columnar flow records: the columns the TAD query selects from the ClickHouse `flows`
 * table (create_table.sh:31-85; anomaly_detection.py:52-61).  IPs are IPv4 packed in host
 * byte order, or host-assigned dictionary ids for anything else (the aggregated-flow
 * modes put their dictionary ids -- podNamespace/podLabels/podName/direction/
 * destinationServicePortName/flowType -- into these same six key slots).  A NULL key
 * column means "all zero".  src_ns/dst_ns are optional namespace dictionary ids used only
 * by the ns_ignore filter (anomaly_detection.py:576-580).
 */
typedef struct {
    uint64_t rows;
    uint64_t capacity;
    int32_t mem;               /* tad_mem: where the column pointers live                           */
    int32_t reserved;
    uint32_t *src_ip;          /* sourceIP                                                          */
    uint32_t *dst_ip;          /* destinationIP                                                     */
    uint16_t *src_port;        /* sourceTransportPort                                               */
    uint16_t *dst_port;        /* destinationTransportPort                                          */
    uint8_t *proto;            /* protocolIdentifier                                                */
    uint32_t *flow_start;      /* flowStartSeconds (DateTime, seconds)                              */
    uint32_t *flow_end;        /* flowEndSeconds                                                    */
    uint64_t *value;           /* throughput (UInt64)                                               */
    uint32_t *src_ns;          /* optional                                                          */
    uint32_t *dst_ns;          /* optional                                                          */
} tad_columns;

/* Job description = the argv the controller builds (controller.go:530-623) after its own
 * validation, with strings already mapped to ids by the host shim. */
typedef struct {
    int32_t algo;              /* tad_algo         --algo                                           */
    int32_t reducer;           /* tad_reducer      implied by --agg-flow                            */
    uint32_t start_time;       /* --start_time as epoch seconds, 0 = unbounded: flow_start >= start */
    uint32_t end_time;         /* --end_time, 0 = unbounded: flow_end < end                         */
    uint32_t flags;            /* TAD_FLAG_*                                                        */
    uint32_t n_ns_ignore;      /* --ns-ignore-list mapped to namespace ids                          */
    const uint32_t *ns_ignore;
    char id[40];               /* --id (uuid, 36 chars + NUL)                                       */
    uint64_t global_rows;      /* world_size > 1: rows of the whole table over all ranks (the host  */
                               /* knows it from its SELECT count()); every rank must pass the same   */
                               /* value.  0 = the ranks agree on it with a blocking all-gather at    */
                               /* job start.  Ignored on a single GPU.                               */
} tad_job_spec;

enum {
    TAD_PHASE_H2D = 0,         /* host -> device copy of the columns (host-resident input only)     */
    TAD_PHASE_HIST,            /* key pack + hash + bucket histogram                                */
    TAD_PHASE_SCAN,            /* bucket offsets                                                    */
    TAD_PHASE_SCATTER,         /* hash partition into 32-byte packed rows                           */
    TAD_PHASE_EXCHANGE,        /* multi-GPU: exposed part of the NCCL all-to-all (exact partition), or the  */
                               /* peer counter gather (optimistic partition: rows are pulled inside GROUP)  */
    TAD_PHASE_GROUP,           /* per-bucket group + time sort + reduce -> per-series arrays        */
    TAD_PHASE_SPILL,           /* oversized buckets through the global-memory path                  */
    TAD_PHASE_DETECT,          /* stddev_samp + EWMA/ARIMA/DBSCAN + anomaly compaction              */
    TAD_PHASE_D2H,             /* result rows device -> host                                        */
    TAD_PHASE_SYNC,            /* multi-GPU: time spent waiting for the other ranks at the job's     */
                               /* barriers (arrival skew + barrier latency; 0 on one GPU)            */
    TAD_NPHASES
};

/* = ThroughputAnomalyDetectorStatus (types.go:114-122) + counters. */
typedef struct {
    int32_t state;             /* tad_state                                                         */
    int32_t completed_stages;  /* maps onto Status.CompletedStages (controller.go:426-453)          */
    int32_t total_stages;      /* maps onto Status.TotalStages                                      */
    int32_t error;             /* tad_error when state == FAILED                                    */
    char err_msg[256];         /* Status.ErrorMsg                                                   */
    uint64_t rows_in;          /* rows handed in (this rank)                                        */
    uint64_t rows_kept;        /* after the stage-A filters (this rank, before exchange)            */
    uint64_t rows_owned;       /* rows this rank owns after the exchange                            */
    uint64_t points;           /* after the stage-A reduce                                          */
    uint64_t series;           /* distinct keys owned by this rank                                  */
    uint64_t result_rows;      /* anomalous points (all points with TAD_FLAG_EMIT_ALL)              */
    uint64_t spill_rows;       /* rows that went through the oversized-bucket path                  */
    uint64_t gpu_launches;     /* kernels of this library launched for the job                      */
    double device_ms;          /* first kernel start -> last kernel end (CUDA events)               */
    double total_ms;           /* submit -> results on host (wall clock)                            */
    double phase_ms[TAD_NPHASES];
} tad_status;

/* Result rows = the columns the reference appends to default.tadetector
 * (anomaly_detection.py:385-393; create_table.sh:363-384), structure-of-arrays, host
 * memory owned by the job, valid until tad_release().  aggType / algoType / id /
 * anomaly="true" are per-job constants the host shim adds, as is the
 * "NO ANOMALY DETECTED" sentinel row when rows == 0 (anomaly_detection.py:395-420). */
typedef struct {
    uint64_t rows;
    const uint32_t *src_ip;
    const uint32_t *dst_ip;
    const uint16_t *src_port;
    const uint16_t *dst_port;
    const uint8_t *proto;
    const uint32_t *flow_start;
    const uint32_t *flow_end;
    const double *stddev;      /* throughputStandardDeviation; NaN = SQL NULL (series of 1 point)   */
    const double *algo_calc;   /* algoCalc                                                          */
    const double *throughput;  /* throughput as Float64                                             */
    const uint8_t *anomaly;    /* 1 = anomalous (always 1 without TAD_FLAG_EMIT_ALL)                */
} tad_rows;

/* Replaces: cluster validation + Spark session bring-up (controller.go:499-503;
 * anomaly_detection.py:651).  Creates streams, NCCL communicator (world_size > 1). */
int tad_init(const tad_config *cfg, tad_ctx **out);
void tad_shutdown(tad_ctx *ctx);

/* Replaces: the JDBC read target (anomaly_detection.py:655-662).  Allocates library-owned
 * pinned host (mem = TAD_MEM_HOST) or device (TAD_MEM_DEVICE) column buffers. */
int tad_alloc_columns(tad_ctx *ctx, uint64_t capacity, int32_t mem, tad_columns *cols);
/* Adds the two optional namespace-id columns (src_ns, dst_ns) to buffers obtained from
 * tad_alloc_columns; needed only when the job carries an ns_ignore list (anomaly_detection.py:576-580). */
int tad_alloc_ns_columns(tad_ctx *ctx, tad_columns *cols);
int tad_free_columns(tad_ctx *ctx, tad_columns *cols);

/* Replaces: CreateSparkApplication (controller.go:685, pkg/controller/util.go:223-233).
 * Non-blocking: validates, enqueues, returns a job handle in state SCHEDULED. */
int tad_submit(tad_ctx *ctx, const tad_job_spec *spec, const tad_columns *cols, tad_job **out);

/* Replaces: GetSparkApplication + Spark-UI stage scraping (controller.go:426-497). */
int tad_poll(tad_job *job, tad_status *status);
/* Convenience: block until COMPLETED/FAILED or timeout_ms (<0 = forever) elapses. */
int tad_wait(tad_job *job, int64_t timeout_ms, tad_status *status);

/* Replaces: SELECT ... FROM tadetector WHERE id = ? (rest.go:249-315) for a finished job. */
int tad_result(tad_job *job, tad_rows *rows);

/* Replaces: DeleteSparkApplication (controller.go:385-424).  tad_cancel returns at once; the job then fails with
 * TAD_ERR_CANCELLED at its next check.  An ARIMA job on one GPU checks inside its fit kernel: every warp stops at its
 * next evaluation round and drops the fits in flight, so the job stops within one likelihood evaluation of the longest
 * prefix being fitted, whatever the series' length (within one phase of the pipeline otherwise).  An ARIMA job whose fit
 * is parked while other jobs run (tad_set_fit_sharing) fails once the job running in its place has ended; its parked
 * buffers are then freed.
 * Several GPUs (world_size > 1): call it on any one rank; the job then fails with TAD_ERR_CANCELLED on every rank, its
 * err_msg naming the rank that cancelled, and no rank is ever left waiting in a collective.  The ranks decide at points
 * they reach together -- the end of the job, or of the current pass under a memory budget -- on what every rank brings
 * there.  An ARIMA fit stops within one evaluation round on every rank when the ranks map each other's memory (the
 * default), otherwise on the cancelling rank only, and the others at the end of their fits.  A cancel that arrives after
 * the rank has reached the job's last such point while no peer is still fitting changes nothing: the job completes on
 * every rank.  A job cancelled in the queue still meets its peers once.
 * tad_release of a job that has not finished cancels it (on several GPUs as above, failing the job on every rank) and
 * waits until it has failed (for a parked ARIMA job, at most the run time of the job running in its place; when that is a
 * streamed ARIMA job fitting beside it, until that job's input has ended and its result is published); the context then
 * runs the next queued job. */
int tad_cancel(tad_job *job);
int tad_release(tad_job *job);

/* Replaces: nothing finer than GetSparkAppProgress's completed / total stages (pkg/controller/util.go:129-159), which
 * tad_poll reports; this counts the work inside the stages, so a long ARIMA fit phase shows that it moves.  Any state,
 * any thread, like tad_poll.  Non-ARIMA jobs: fits 0 / 0.  The counts never decrease, except that a pass which is split
 * after its fit phase gives its fits back. */
typedef struct {
    uint32_t passes_done;   /* hash-range passes whose pipeline has finished                          */
    uint32_t passes;        /* passes planned so far (grows when a pass splits)                        */
    uint64_t fits_done;     /* ARIMA prefix fits finished, summed over the passes so far               */
    uint64_t fits_total;    /* ARIMA prefix fits of the passes whose fit phase has started              */
} tad_progress;
int tad_job_progress(tad_job *job, tad_progress *p);

/* Device memory this context's workspace may hold (bytes).  0 (default) = what is free on the device when a job starts,
 * plus what the context already holds, less a headroom of 512 MiB.  A job that does not fit runs in hash-range passes:
 * the connections are split by the low bits of their key hash into 2, 4, ... 64 disjoint sets, each run through the
 * whole pipeline; the result rows are the same rows a one-pass run gives.  Host-resident input is read over PCIe once
 * per pass.  A job fails with TAD_ERR_NOMEM only when a 1/64 hash range of it does not fit.  Caller-owned columns and
 * pinned host memory are not counted.  If the budget drops below what the context holds, the workspace is freed before
 * the next job.  Applies to jobs that start after the call; TAD_ERR_INVALID_ARG below the floor of 64 MiB.  With fit
 * sharing on (tad_set_fit_sharing), an ARIMA tad_submit job, or a streamed one with TAD_FLAG_SHARE, plans in this budget
 * less the reserve (TAD_ERR_NOMEM when that is below 64 MiB), and the jobs run beside its fit plan in the reserve.
 *
 * Several GPUs (world_size > 1): 0 means "no planning", not free memory: a job without a budget runs exactly as it does
 * without this call (no planning collective, launch or sync).  With one, the ranks run the same passes over their shards
 * at once: they agree on the pass count from every rank's rows and budget (one blocking all-gather at job start) and the
 * first sweep's per-owner counts, and every pass ends with an 8-byte all-gather on which they split it or stop together.
 * The ranks may set different values, each rank's workspace staying inside its own, but every rank of a job must have a
 * nonzero budget or none (like the run-time switches every rank must see alike).  The job fails with TAD_ERR_NOMEM on
 * every rank, naming the rank and the bytes, when a 1/64 hash range does not fit one rank, and a tad_cancel on any rank
 * fails the job with TAD_ERR_CANCELLED on every rank, at the end of the current pass (a job cancelled before it started
 * still meets its peers once).  The contexts stay usable in both cases.  The exported partition buffer of earlier jobs is
 * freed at the start of such a job.  Host or device columns as for tad_submit; streamed input as under "Several GPUs" below. */
int tad_set_memory_budget(tad_ctx *ctx, uint64_t bytes);
/* For a COMPLETED job: the passes it ran in (the same count on every rank of a multi-GPU job) and the largest device
 * workspace the context held while it ran (TAD_ERR_STATE otherwise). */
int tad_job_memory(tad_job *job, uint32_t *passes, uint64_t *peak_workspace_bytes);

/* Fit sharing (single GPU).  A context runs its jobs one at a time, and an ARIMA job's fit phase can take minutes: without
 * sharing, every job submitted meanwhile waits for it.  reserve_bytes = 0 (default): off, jobs run strictly in submit order.
 * Nonzero: an ARIMA tad_submit job plans its passes in the memory budget less `reserve_bytes`, and while its fit runs, an
 * EWMA or DBSCAN tad_submit job in the queue makes the fit yield within one evaluation round.  The fit's device buffers
 * are then parked (kept, the rest of its workspace freed), the EWMA and DBSCAN tad_submit jobs queued at that moment run
 * in submit order with the reserve as their memory budget (in hash-range passes if need be), and the fit resumes where
 * it stopped.  Its forecasts, rows and fit counts are those of an uninterrupted run.  A queued job whose 1/64 hash range
 * does not fit the reserve is not failed: that is found out by running it in the reserve (its first sweep reads its
 * input; it shows RUNNING, then SCHEDULED again with its stages and progress back at 0), and it then waits for its
 * turn, as without sharing.  A yield drops the fits in flight, which the resume fits again; the fit does not yield again
 * until all of them have finished and it has run at least as long as the jobs run in its place took, so no fit is
 * dropped twice and a steady stream of short jobs at most about doubles its fit phase.  The ARIMA job's device_ms and
 * detect phase leave out the time it was parked (tad_job_yields); its tad_job_memory peak leaves out the workspace of the
 * jobs run in its place, theirs leaves out its parked buffers and stays within the reserve, so the two stay inside the
 * budget.  Applies to jobs that start after the call.
 *
 * Streamed jobs (tad_submit_stream, tad_submit_stream_filtered) take part only with TAD_FLAG_SHARE in their spec's flags;
 * without it a streamed job neither yields nor runs in a yield, as with sharing off.  The flag is ignored on tad_submit
 * jobs, which take part anyway, and on a context whose sharing is off.  A streamed ARIMA job with the flag plans in the
 * budget less the reserve and its fit yields as above: its text key dictionaries, its round in progress and its host
 * row store pages are kept while it is parked, and its feeder's pending push or end call goes on with the same round.  A
 * streamed EWMA or DBSCAN job with the flag runs in a yield only once its feeder has pushed its first block (or ended
 * its round): a job whose caller has not started delivering never parks a fit.  It then runs in the reserve as the
 * others do, with its own dictionaries and as many rounds as it needs, and its caller's blocks are taken meanwhile; the
 * fit stays parked until its input has ended and its result is published.  Its host row store use stays within the host
 * budget less the pages the parked job holds; without room it asks for rounds, as a job without a store does.  If it
 * does not fit the reserve, the round it was running in is read to its end without being used and its tad_stream_end
 * returns *again = 1; the job is SCHEDULED again with its stages and progress at 0, is not run in a yield again, and
 * its next round's blocks are taken once the context reaches the job in its turn, which starts it again from its first
 * round.
 *
 * An ARIMA tad_submit job with TAD_FLAG_FIT_BESIDE may run in a yield too, and fits beside the yielded fit instead of
 * waiting for it: one such job per yield, the first queued, while the yielded job's reserve is at least 128 MiB.  It
 * plans in half the reserve and keeps the other half as its own reserve, so its fit yields in turn to the EWMA and DBSCAN
 * jobs queued meanwhile, which run in that half.  Its fit runs in one launch with the rest of the yielded fit, each with
 * about half the GPU; once all its fits are done the launch ends within one evaluation round (after the yielded fit has
 * finished again the fits its yield dropped), its rows are scored and it completes, and the yielded fit resumes as after
 * any yield.  Every job's forecasts, rows and fit counts are those of a solo run.  A job whose 1/64 hash range does not
 * fit half the reserve waits for its turn as above.  A cancel of the flagged job ends the joint launch; a cancel of the
 * yielded job stops its part at once and takes effect once the flagged job has ended.  The yielded job's detect phase and
 * device_ms count its time in the joint launch as fit time; its tad_job_memory peak leaves out the flagged job's
 * workspace, whose own peak stays within half the reserve.
 *
 * A streamed ARIMA job fits beside a yielded fit under the same rules when its spec carries both TAD_FLAG_SHARE and
 * TAD_FLAG_FIT_BESIDE (either flag alone leaves it waiting for its turn), and, like a streamed EWMA or DBSCAN job, only
 * once its feeder has pushed its first block or ended its round.  Its passes each fit in one launch with the rest of the
 * yielded fit; between them the yielded fit stays parked while its caller delivers further rounds (without a host row
 * store), and its store pages come from the host budget less every page held, as above.  If it does not fit half the
 * reserve (a 1/64 hash range, or its text key dictionaries), its round ends with *again = 1 and it waits for its turn as
 * above.  A cancel of it ends the joint launch, and its feeder's pending push or end call returns TAD_ERR_CANCELLED.  A
 * cancel of the yielded job takes effect once the streamed job's input has ended and its result is published; a
 * tad_release of the yielded job waits that long too.
 *
 * Lending (TAD_FLAG_LEND).  A streamed job holds the context while its worker waits for the caller's next block, and
 * the caller's source (a ClickHouse SELECT) is usually far slower than the GPU.  A streamed job (tad_submit_stream,
 * _filtered, _filtered_ns) with TAD_FLAG_LEND, started while sharing is on, plans in the budget less the reserve (its
 * text key dictionaries grow inside that amount) and lends the GPU while it waits: when no block is pending and its
 * round has not ended (before the first block, between blocks, before tad_stream_end, between rounds), the wait has
 * lasted a few milliseconds and an EWMA or DBSCAN tad_submit job is queued.  Its workspace is then parked as a yielded
 * fit's is, the blocks it has taken are released, and the EWMA and DBSCAN tad_submit jobs queued at that moment run in
 * submit order with the reserve as their budget; one whose 1/64 hash range does not fit it is put back, as in a yield.
 * ARIMA and streamed jobs never run in a lend.  Before each job the lend ends if a block is pending, the round has
 * ended or the job is cancelled, so a pushed block waits for at most one lent job.  After a lend the job does not lend
 * again until as much time has passed as the lend took, so under a steady stream of short jobs its own time from the
 * first block to the result at most about doubles.  A job running in a fit's yield or beside a fit does not lend.  A
 * streamed ARIMA job with TAD_FLAG_SHARE | TAD_FLAG_LEND lends while it reads its input and yields while it fits.
 * Every job's rows, text ids, fit counts and pass counts are those of a run without lending.  A cancel of the lending
 * job takes effect once the lent job in progress has ended: its parked buffers are freed and its feeder's pending push
 * or end call returns TAD_ERR_CANCELLED (tad_release waits that long).  The lending job's device_ms and h2d phase leave
 * out the time it was lent (tad_job_lent), its tad_job_memory peak leaves out the lent jobs' workspace, theirs stays
 * within the reserve, and its host row store pages are untouched.
 * TAD_ERR_INVALID_ARG for a nonzero value below 64 MiB; TAD_ERR_UNSUPPORTED when world_size > 1 (a rank whose fit
 * yielded alone would leave its peers waiting for it; the ranks would have to agree on each yield). */
int tad_set_fit_sharing(tad_ctx *ctx, uint64_t reserve_bytes);
/* For a COMPLETED ARIMA job: how many times its fit phase yielded and the time it spent parked (ms).  TAD_ERR_STATE for
 * any other job or state. */
int tad_job_yields(tad_job *job, uint32_t *yields, double *parked_ms);
/* For a COMPLETED streamed job: the number of jobs that ran in its lends (TAD_FLAG_LEND) and the time it was lent (ms),
 * both 0 if it never lent.  TAD_ERR_STATE for any other job or state; TAD_ERR_INVALID_ARG for a NULL argument. */
int tad_job_lent(tad_job *job, uint32_t *jobs_run, double *lent_ms);

/* Pinned host memory this context may hold for its host row store (bytes).  0 (default) = no store.  With a store, a
 * streamed job (tad_submit_stream) that needs more than one hash-range pass keeps its first round's filtered rows in
 * pinned host pages (32 bytes per row) and loads every pass from them, so the caller delivers its rows once whatever the
 * pass count.  If the store would outgrow the budget, or the memory cannot be pinned, the job drops the store and goes on
 * as without one: that round only counts its rows and further rounds are asked for.  tad_submit jobs and streamed jobs
 * that run in one pass never use it.  The context keeps its pages for the next job up to the budget; pages above a
 * lowered budget are freed before the next job, and tad_shutdown frees them all.  Applies to jobs that start after the
 * call: a job reads the budget once, when the context starts running it (for a streamed job on an idle context that is
 * at submit, before its first block).  Single GPU only (TAD_ERR_UNSUPPORTED when world_size > 1); TAD_ERR_INVALID_ARG
 * for a nonzero value below 64 MiB. */
int tad_set_host_budget(tad_ctx *ctx, uint64_t bytes);
/* For a COMPLETED job: the rows that went through the host row store (0 if it was not used) and the most store bytes the
 * context held while the job ran (TAD_ERR_STATE otherwise). */
int tad_job_host_memory(tad_job *job, uint64_t *stored_rows, uint64_t *peak_host_bytes);

/* ---- Streamed input (single GPU) ---------------------------------------------------------------------------------
 * The job's rows arrive as column blocks while it runs (a ClickHouse SELECT hands them over block by block), so the
 * table never has to be in host memory at once and may hold more than 2^32 rows.  A ROUND is one complete delivery of
 * the job's rows, in any order and any block sizes: tad_stream_push each block, then tad_stream_end.  When the job
 * needs more than one hash-range pass (see tad_set_memory_budget), tad_stream_end sets *again = 1 and the caller
 * delivers the same rows again; *again = 0 means the input is complete, and from then on tad_wait / tad_poll /
 * tad_result / tad_job_memory behave as for any job.  Without a host row store there are as many rounds as a host-input
 * job of the same rows makes sweeps over its table.  With one (tad_set_host_budget), a round that went to the store
 * ends with *again = 0: the passes are loaded from the store.
 *
 * Submit: rows_hint is the caller's estimate of one round's rows (its SELECT count()), 0 = unknown.  It only chooses the
 * pass count and sizes the pass columns before the first round: a wrong hint may cost one round more, never a different
 * result.  TAD_ERR_UNSUPPORTED when world_size > 1 without TAD_FLAG_RANK_STREAM.  A context still runs one job at a time: a streamed job holds the
 * worker from when it starts until its input ends, and pushes made before the worker reaches the job wait for it.  The
 * one exception is fit sharing (tad_set_fit_sharing): with TAD_FLAG_SHARE in its spec, a streamed EWMA or DBSCAN job
 * whose caller has pushed its first block may run while an ARIMA fit is parked, and a streamed ARIMA job's fit yields;
 * with TAD_FLAG_FIT_BESIDE as well, a streamed ARIMA job so fed may fit beside a parked fit; with TAD_FLAG_LEND, a
 * streamed job lends the GPU to queued EWMA and DBSCAN tad_submit jobs while it waits for its caller.
 *
 * Blocks: mem is TAD_MEM_HOST (any host memory; pinned buffers from tad_alloc_columns copy at the full PCIe rate) or
 * TAD_MEM_DEVICE (read in place); fewer than 2^32 rows; flow_end and value are required; every block carries the same
 * non-NULL columns as the job's first block (src_ns / dst_ns included).  A block that breaks one of these fails the job
 * with TAD_ERR_INVALID_ARG.  A pushed block must stay valid and unchanged until the next tad_stream_push or
 * tad_stream_end call on the job returns: the caller may fill block k+1 while block k is being copied.
 *
 * Each pass, not the job, must stay below 2^32-2 rows.  When there is more than one round, every round must deliver,
 * after the time-window and ns_ignore filters, as many rows of each low-hash-bit residue as the first round did;
 * otherwise (the source changed between reads, e.g. an open-ended window over a table being appended to) the job fails
 * with TAD_ERR_INVALID_ARG.  This is a check on counts, not on content.
 *
 * Status: rows_in and rows_kept count one round; phase times and device_ms sum over rounds and passes (the h2d phase of
 * a streamed round includes the time the engine waited for its blocks); state is RUNNING while the job waits for input.
 *
 * Errors: push / end on a job not submitted with tad_submit_stream, or after its input is complete: TAD_ERR_STATE.
 * After tad_cancel: TAD_ERR_CANCELLED, and the job is FAILED.  Once the job has failed, its error code.  tad_release of
 * a job whose input has not ended cancels it.  The context stays usable for the next job in every case.
 * tad_shutdown cancels a streamed job that waits for input; as for every job, release it before tad_shutdown.
 *
 * Threads: while the feeding thread is inside tad_stream_push or tad_stream_end, other threads may call tad_poll and
 * tad_cancel on the job, but not tad_release: release it after the feeding thread has returned.
 *
 * Several GPUs (world_size > 1): tad_submit_stream with TAD_FLAG_RANK_STREAM in the spec's flags submits this rank's part
 * of a job whose rows are streamed to every rank; without the flag a rank engine refuses it (TAD_ERR_UNSUPPORTED), and
 * tad_submit_stream_filtered / _filtered_ns with a filter refuse rank engines with or without it (with a NULL filter
 * they are tad_submit_stream).  Every rank submits its part, in the
 * same order relative to its other jobs, as for tad_submit on several GPUs.
 *   Rows: each rank's caller pushes any disjoint share of the table, in any split: rows of one connection may arrive on
 *     any rank, since the owner rank still comes from the key hash.  Every rank's blocks carry the same non-NULL columns
 *     (a rank whose first round is empty carries none and agrees with any); key ids (host dictionary ids) must mean the
 *     same on every rank.  A mismatched column set fails every rank with TAD_ERR_INVALID_ARG.
 *   rows_hint: this rank's own share of one round, 0 = unknown; spec.global_rows is ignored.  As on one GPU, it only
 *     seeds the plan: a wrong hint may cost one round more, never a different result.
 *   Threads: each rank is fed from its own thread or process.  tad_stream_end returns once every rank has ended the
 *     round, and its *again is the same on every rank: the ranks decide it from all-gathered counts.  A rank whose caller
 *     stops delivering without ending its round holds its peers at the round's end until someone cancels the job.
 *   Rounds: every later round must deliver, on every rank, the per-residue counts that rank's first round delivered;
 *     otherwise every rank fails with TAD_ERR_INVALID_ARG, its err_msg naming the rank.
 *   Budget: a rank stream job always plans, as a single-GPU streamed job does, in tad_set_memory_budget or, when that is
 *     0, the free device memory less a 512 MiB headroom, each rank in its own.  (The "0 = no planning" rule of rank
 *     tad_submit jobs is unchanged.)  A 1/64 hash range that does not fit one rank fails every rank with TAD_ERR_NOMEM.
 *   Cancel: tad_cancel on any rank makes that rank's pending and later push or end calls return TAD_ERR_CANCELLED at
 *     once; its engine treats the rest of the round as empty and still meets its peers.  The job fails with
 *     TAD_ERR_CANCELLED on every rank: within one block on the peers where the ranks map each other's stop board (the
 *     default), and their pending push or end calls return TAD_ERR_CANCELLED too; otherwise at the end of the round.
 *     tad_release of a rank job whose input has not ended cancels it the same way.
 *   Refused or ignored: tad_stream_push_text and _text_ns return TAD_ERR_UNSUPPORTED, and the job fails with it on every
 *     rank at the round's end.  TAD_FLAG_SHARE, TAD_FLAG_FIT_BESIDE and TAD_FLAG_LEND are ignored (fit sharing is single
 *     GPU), and there is no host row store (tad_set_host_budget is single GPU). */
int tad_submit_stream(tad_ctx *ctx, const tad_job_spec *spec, uint64_t rows_hint, tad_job **out);
/* Hands one block of the current round to the job; returns once the engine has finished reading the previous block. */
int tad_stream_push(tad_job *job, const tad_columns *block);
/* Closes the round; returns once the engine has finished with the round's rows, with *again = 1 when the same rows
 * must be pushed again for another pass, 0 when the input is complete.  again may be NULL. */
int tad_stream_end(tad_job *job, int32_t *again);

/* ---- Text key slots of streamed blocks ---------------------------------------------------------------------------
 * Replaces: the host dictionary pass over sourceIP / destinationIP String columns (create_table.sh:38-39) that turns
 * IPv6 and other non-IPv4 text into key ids before tad_stream_push.  A text column is a Native String column exactly as
 * it sits in the block: `rows` x (VarUInt length, bytes), `nbytes` long, and marks[k] = the byte offset of row 32k
 * (ceil(rows / 32) marks, marks[0] = 0).  The engine decodes it and dictionary-encodes it on the GPU into job-stable u32
 * ids, dense and in order of first appearance (over the round's rows, in push order, then row order: the ids a host
 * dictionary built the same way gives), so every round and pass of a job keys the same name alike.  The dictionary and
 * the text staging count against tad_set_memory_budget and in tad_job_memory's peak; a first round whose dictionary
 * leaves no room for its pass columns only counts its rows (one more round is asked for), and a dictionary that does not
 * fit by itself fails the job with TAD_ERR_NOMEM. */
typedef struct {
    const uint8_t *bytes;      /* the column's bytes (host memory)                                                   */
    uint64_t nbytes;
    const uint64_t *marks;     /* ceil(rows / 32) byte offsets: of rows 0, 32, 64, ...                               */
} tad_text_column;
/* tad_stream_push with src_ip / dst_ip given as text: a NULL text pointer means that slot comes from `block` as for
 * tad_stream_push; a slot given as text must have its u32 column NULL.  Which slots are text is part of the job's column
 * set: every block must make its first block's choice.  Text is accepted in host blocks (mem = TAD_MEM_HOST) only.  A
 * block that breaks one of these, marks that decrease or pass nbytes, or (found on the GPU, reported by this call or a
 * later push / end call) VarUInt lengths that do not end exactly at the next mark fail the job with
 * TAD_ERR_INVALID_ARG.  TAD_ERR_UNSUPPORTED for a job not submitted with tad_submit_stream (tad_submit_stream itself is
 * single-GPU only).  The block and its text columns must stay valid and unchanged until the next push or end call
 * returns.  Errors and threads otherwise as for tad_stream_push. */
int tad_stream_push_text(tad_job *job, const tad_columns *block, const tad_text_column *src_ip,
                         const tad_text_column *dst_ip);
/* For a COMPLETED job: the dictionary of text slot `slot` (0 = src_ip, 1 = dst_ip): the name of id k is
 * bytes[offsets[k] .. offsets[k + 1]), *count names, in host memory owned by the job until tad_release.
 * TAD_ERR_STATE before completion and for a slot the job did not take as text.  Any thread. */
int tad_job_names(tad_job *job, int32_t slot, const uint8_t **bytes, const uint64_t **offsets, uint32_t *count);

/* ---- Row predicates of a streamed job's text slots ---------------------------------------------------------------
 * Replaces: the String predicates of the aggregated-flow queries (anomaly_detection.py:566-609), which the host can no
 * longer apply once a block hands its String key columns over as text.  The engine evaluates them on the GPU, once per
 * distinct name while the first round builds the dictionaries, and drops the rows that fail:
 *   TAD_NAME_ANY        every name                                                      (no predicate on the slot)
 *   TAD_NAME_EQ         the name's bytes equal the pattern's                  podName = x, podNamespace = x (:566-575),
 *                                                                             destinationServicePortName = x (:598-602),
 *                                                                             destinationIP = x (:590-592)
 *   TAD_NAME_NONEMPTY   a name of length > 0                                  podLabels <> '' (:577-578),
 *                                                                             destinationServicePortName <> '' (:603-604)
 *   TAD_NAME_ICONTAINS  pattern.lower() in name.lower(), as Python has it     ilike(podLabels, '%x%') (:560-565), with
 *                       for a UTF-8 name and an ASCII pattern: A-Z fold to    '%' and '_' in x taken literally, as the
 *                       a-z; U+0130 (C4 B0) folds to 'i' followed by          host mirror takes them
 *                       U+0307, U+212A (E2 84 AA) to 'k' (the only two non-ASCII code points that lower-case to ASCII);
 *                       every other byte compares exactly.  A pattern byte >= 0x80 is TAD_ERR_INVALID_ARG at submit.
 *   proto_eq            -1 = none; 0..255: keep only rows whose proto byte equals it    flowType = 3 (:587-589)
 * A row is kept when every slot's predicate holds for its name, proto_eq holds, and the time-window and ns_ignore filters
 * hold.  Dropped rows count as filtered: rows_kept, the per-residue round-consistency counts and the host row store see
 * only kept rows.  The dictionaries still hold every name of the job's rows (tad_job_names), kept or not.
 *
 * TAD_ERR_INVALID_ARG, the context usable afterwards in every case: at submit for a bad op, a NULL pattern with a nonzero
 * length, an ICONTAINS pattern byte >= 0x80 or proto_eq outside -1..255 (the job is returned FAILED); at the first push
 * (the job fails) for a predicate on a slot the first block does not give as text, or proto_eq without a proto column or
 * without any text slot.  Single GPU and host blocks only, as for tad_stream_push_text. */
enum { TAD_NAME_ANY = 0, TAD_NAME_EQ = 1, TAD_NAME_NONEMPTY = 2, TAD_NAME_ICONTAINS = 3 };
typedef struct {
    int32_t op[2];              /* per text slot (0 = src_ip, 1 = dst_ip): TAD_NAME_*                                    */
    const uint8_t *pattern[2];  /* EQ / ICONTAINS; copied by the call                                                    */
    uint32_t pattern_len[2];
    int32_t proto_eq;           /* -1 = none; 0..255: keep only rows whose proto byte equals it                          */
} tad_stream_filter;
/* tad_submit_stream with row predicates; a NULL filter is tad_submit_stream. */
int tad_submit_stream_filtered(tad_ctx *ctx, const tad_job_spec *spec, uint64_t rows_hint, const tad_stream_filter *filter,
                               tad_job **out);

/* ---- Namespace ignore list on namespace text ---------------------------------------------------------------------
 * Replaces: sourcePodNamespace NOT IN (...) AND destinationPodNamespace NOT IN (...) (anomaly_detection.py:576-580) for a
 * streamed job whose blocks hand their namespace columns over as Native String text (tad_stream_push_text_ns), so that
 * no namespace column is dictionary-encoded on the host.  The list is given as names; the engine tests every row's
 * namespace against it on the GPU, in every round and pass:
 *   - a name is listed when its bytes equal a listed name's bytes exactly (no case folding, no trimming, no Unicode
 *     normalisation: the reference's NOT IN compares String bytes);
 *   - the empty namespace is a name like any other: it is dropped only when "" is in the list;
 *   - a row is dropped when its source or its destination namespace is listed (a slot the block does not carry is
 *     never listed);
 *   - a dropped row counts as filtered everywhere a time-window or ns_ignore filter does: rows_kept, the per-residue
 *     round-consistency counts and the host row store see only kept rows.
 * An empty list drops nothing, and the namespace text is then not read.  At most 1024 names of at most 32 KiB in all.
 * A job that pushes namespace text gives its list here and spec->n_ns_ignore = 0; a job that pushes u32 namespace ids
 * keeps spec->ns_ignore as before and gives no names here. */
typedef struct {
    tad_stream_filter rows;        /* the text slots' row predicates, as for tad_submit_stream_filtered                */
    uint32_t n_ns_ignore;          /* --ns-ignore-list as names                                                        */
    const uint8_t *ns_ignore_bytes;    /* the names back to back; copied by the call                                  */
    const uint64_t *ns_ignore_offsets; /* n_ns_ignore + 1 offsets from 0: name k is bytes[offsets[k] .. offsets[k + 1])*/
} tad_stream_filter_ns;
/* tad_submit_stream_filtered with the ignore list as names.  TAD_ERR_INVALID_ARG at submit (the job is returned FAILED)
 * for what tad_submit_stream_filtered rejects, offsets that do not start at 0 or decrease, NULL bytes or offsets with a
 * nonzero count, a list over the limits above, or names given together with spec->n_ns_ignore != 0.  A NULL filter is
 * tad_submit_stream. */
int tad_submit_stream_filtered_ns(tad_ctx *ctx, const tad_job_spec *spec, uint64_t rows_hint,
                                  const tad_stream_filter_ns *filter, tad_job **out);
/* tad_stream_push_text with src_ns / dst_ns given as text too (tad_text_column: the column's bytes and the offset of
 * every 32nd row), any of the four pointers NULL.  A namespace slot given as text must have its u32 column NULL in
 * `block`, and a block gives its namespace columns either all as text or all as u32 ids.  Which slots are text is part
 * of the job's column set: every block must make its first block's choice.  A job whose first block gives namespace
 * text must have no spec->ns_ignore ids; a job with ignore-list names must not give its namespace columns as ids.  Host
 * blocks only.  The namespace text is staged, cut at marks and counted in the memory budget with the address text; it
 * needs no dictionary.  A block that breaks one of these, marks that decrease or pass nbytes, or (found on the GPU,
 * reported by this call or a later push / end call) VarUInt lengths that do not end exactly at the next mark fail the
 * job with TAD_ERR_INVALID_ARG; the context stays usable.  Otherwise as tad_stream_push_text, which is this call with
 * src_ns = dst_ns = NULL. */
int tad_stream_push_text_ns(tad_job *job, const tad_columns *block, const tad_text_column *src_ip,
                            const tad_text_column *dst_ip, const tad_text_column *src_ns, const tad_text_column *dst_ns);

const char *tad_strerror(int err);
int tad_abi_version(void);

/* Multi-GPU bring-up: rank 0 obtains a 128-byte ncclUniqueId here, the host distributes it
 * (the Go shim over its own channel, bench.py over torch.distributed) and every rank passes
 * it to tad_init.  Replaces: Spark's driver/executor rendezvous (no reference call site). */
int tad_get_unique_id(void *out, size_t bytes);

/* ---- ClickHouse Native-format helpers (host only: no GPU, no context) -----------------------------------------
 * The reference job moves rows over JDBC (read: anomaly_detection.py:655-662; write: :713-726).  The shim streams
 * `SELECT ... FORMAT Native` column blocks instead (clickhouse-go, go.mod:7) and copies every fixed-width column
 * (UInt8/16/64, DateTime = UInt32; create_table.sh:31-85) straight into the tad_columns buffers.  Only String
 * columns need work: these calls index them, turn IPv4 text into the u32 key column and back, and dictionary-encode the rest.
 * theia_b200/clickhouse_native.py is the block reader / writer built on them. */

/* A String column of `rows` values is rows x (VarUInt length, bytes).  Writes the payload position and length of
 * every value and the number of bytes consumed.  TAD_ERR_INVALID_ARG if the buffer ends early or a length >= 2^32. */
int tad_ch_string_index(const uint8_t *buf, size_t len, uint64_t rows, uint64_t *offsets, uint32_t *lengths,
                        size_t *consumed);
/* "a.b.c.d" -> a<<24 | b<<16 | c<<8 | d.  is_v4[i] = 0 (and out[i] = 0) for anything else (IPv6, empty, names):
 * the caller gives those rows dictionary ids.  sourceIP / destinationIP are String columns (create_table.sh:38-39). */
int tad_ch_parse_ipv4(const uint8_t *buf, const uint64_t *offsets, const uint32_t *lengths, uint64_t rows,
                      uint32_t *out, uint8_t *is_v4);
/* u32 -> String column bytes (VarUInt length + "a.b.c.d" per row) for the tadetector INSERT (create_table.sh:363-384).
 * Needs at most 16 bytes per row; TAD_ERR_INVALID_ARG if out_cap is too small. */
int tad_ch_format_ipv4(const uint32_t *ips, uint64_t rows, uint8_t *out, size_t out_cap, size_t *written);
/* Dictionary ids -> String column bytes (VarUInt length + name per row) for the tadetector INSERT, the name of id k being
 * bytes[offsets[k] .. offsets[k + 1]) (tad_job_names).  TAD_ERR_INVALID_ARG for an id >= count or when out_cap is too
 * small; *written = the bytes written. */
int tad_ch_format_names(const uint8_t *bytes, const uint64_t *offsets, uint32_t count, const uint32_t *ids, uint64_t rows,
                        uint8_t *out, size_t out_cap, size_t *written);

/* Dense dictionary ids (order of first appearance) for a String column: ids[i] in [0, *n_unique); first_row[k] is the
 * row at which id k first occurs (the caller reads the k-th name from there).  first_row needs room for `rows` entries.
 * This is how pod namespaces / labels / service-port names become the u32 key columns of the aggregated-flow modes
 * (anomaly_detection.py:511-609) and the namespace ids of the ignore list (:576-580). */
int tad_ch_dictionary(const uint8_t *buf, const uint64_t *offsets, const uint32_t *lengths, uint64_t rows, uint32_t *ids,
                      uint64_t *first_row, uint32_t *n_unique);

#ifdef __cplusplus
}
#endif
#endif /* THEIA_TAD_H */
