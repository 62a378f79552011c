// Host side of the TAD engine: C ABI (include/theia_tad.h), job queue, workspace, phase
// orchestration.  One worker thread per context runs jobs FIFO on one CUDA stream; callers
// (the controller's workers, pkg/controller/util.go:43) only enqueue and poll.
#include <algorithm>
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <deque>
#include <mutex>
#include <thread>
#include <vector>

#include <sched.h>
#include <sys/syscall.h>
#include <unistd.h>

#include "../../include/theia_tad.h"
#include "tad_kernels.h"
#include "tad_nccl.h"
#include "tad_text.h"

using namespace tad;

namespace {

struct DevBuf {
    void *p = nullptr;
    size_t cap = 0;
};

struct PinnedBlock {
    void *p = nullptr;
    size_t cap = 0;
};

constexpr int kMaxEvents = 24;
constexpr int kMaxChunks = 16;          // host-resident input is copied and histogrammed in chunks
constexpr int kMaxRanks = 8;      // also the stop board's words, all of which the multi-GPU fit kernel reads (StopBoard)
static_assert(kMaxRanks == 8, "the fit kernel reads the stop board as 8 words");
constexpr int kMaxXChunks = kMaxSeg / kMaxRanks;   // exchange chunks: scatter of chunk c+1 overlaps the all-to-all of chunk c
constexpr int kTotalStages = 6;   // ingest, partition, exchange, group, detect, egress

// ---- NUMA placement of pinned host memory --------------------------------------------------------------------------
// On a two-socket box half of the GPUs hang off each socket; a pinned buffer on the wrong socket makes every H2D / D2H
// copy cross the inter-socket link, and eight ranks doing that at once is what held the 8-GPU end-to-end rate down in
// round 1.  Pinned allocations therefore happen with the calling thread temporarily confined to the CPUs of the GPU's
// NUMA node (the driver touches the pages inside cudaHostAlloc: first touch = local), with a PREFERRED memory policy on
// top where the container allows set_mempolicy.  TAD_NUMA=0 switches all of it off.
struct NumaInfo {
    int node = -1;
    cpu_set_t cpus;
    bool ok = false;
};

NumaInfo numa_of_device(int device)
{
    NumaInfo ni;
    CPU_ZERO(&ni.cpus);
    if (const char *e = getenv("TAD_NUMA")) if (atoi(e) == 0) return ni;
    char bus[32] = {0};
    if (cudaDeviceGetPCIBusId(bus, sizeof(bus), device) != cudaSuccess) { cudaGetLastError(); return ni; }
    for (char *p = bus; *p; p++) if (*p >= 'A' && *p <= 'Z') *p = (char)(*p - 'A' + 'a');
    char path[128];
    snprintf(path, sizeof(path), "/sys/bus/pci/devices/%s/numa_node", bus);
    FILE *f = fopen(path, "r");
    if (!f) return ni;
    int node = -1;
    if (fscanf(f, "%d", &node) != 1) node = -1;
    fclose(f);
    if (node < 0) return ni;
    snprintf(path, sizeof(path), "/sys/devices/system/node/node%d/cpulist", node);
    f = fopen(path, "r");
    if (!f) return ni;
    char list[4096] = {0};
    if (!fgets(list, sizeof(list), f)) list[0] = 0;
    fclose(f);
    int n = 0;
    for (char *p = list; *p && *p != '\n';) {          // "0-31,64-95"
        char *end = nullptr;
        long a = strtol(p, &end, 10), b = a;
        if (end == p) break;
        if (*end == '-') { p = end + 1; b = strtol(p, &end, 10); }
        for (long c = a; c <= b && c < CPU_SETSIZE; c++) { CPU_SET((int)c, &ni.cpus); n++; }
        p = *end == ',' ? end + 1 : end;
    }
    // only CPUs this process may use anyway
    cpu_set_t allowed;
    if (sched_getaffinity(0, sizeof(allowed), &allowed) == 0) {
        n = 0;
        for (int c = 0; c < CPU_SETSIZE; c++) {
            if (CPU_ISSET(c, &ni.cpus) && !CPU_ISSET(c, &allowed)) CPU_CLR(c, &ni.cpus);
            if (CPU_ISSET(c, &ni.cpus)) n++;
        }
    }
    ni.node = node;
    ni.ok = n > 0;
    return ni;
}

// Scope guard: the calling thread runs on (and prefers memory of) the GPU's NUMA node while it is alive.
struct NumaScope {
    cpu_set_t saved;
    bool restore = false, policy = false;
    explicit NumaScope(const NumaInfo &ni)
    {
        if (!ni.ok) return;
        if (sched_getaffinity(0, sizeof(saved), &saved) != 0) return;
        if (sched_setaffinity(0, sizeof(ni.cpus), &ni.cpus) == 0) restore = true;
#ifdef SYS_set_mempolicy
        unsigned long mask[16] = {0};
        if (ni.node < (int)(sizeof(mask) * 8)) {
            mask[ni.node / (8 * sizeof(unsigned long))] |= 1ul << (ni.node % (8 * sizeof(unsigned long)));
            policy = syscall(SYS_set_mempolicy, 1 /* MPOL_PREFERRED */, mask, sizeof(mask) * 8) == 0;
        }
#endif
    }
    ~NumaScope()
    {
#ifdef SYS_set_mempolicy
        if (policy) syscall(SYS_set_mempolicy, 0 /* MPOL_DEFAULT */, nullptr, 0);
#endif
        if (restore) sched_setaffinity(0, sizeof(saved), &saved);
    }
};

double now_ms()
{
    using namespace std::chrono;
    return duration<double, std::milli>(steady_clock::now().time_since_epoch()).count();
}

}  // namespace

// The fit of an ARIMA pass, as its wait (wait_fit) and its yields see it.  While the pass is parked its buffers stay in
// device memory, so a flagged ARIMA job run in its yield fits beside it (ctx->beside) from its part alone.
struct YieldedFit {
    tad_job *job;
    FitPart part;                    // its series, buffers, words and resume points
    uint64_t done0 = 0, total0 = 0;  // its fit counts before the pass (tad_job_progress adds the pass's counters to them)
    uint32_t dropped = 0;            // fits its last leave dropped: the next launch it takes part in redoes them
    double fit_ms = 0;               // time its part spent in joint launches since the yield: fit time, not parked time
};

struct tad_job {
    tad_ctx *ctx = nullptr;
    tad_job_spec spec{};
    std::vector<uint32_t> ns_ignore;
    tad_columns cols{};
    std::mutex mu;
    std::condition_variable cv;
    tad_status st{};
    std::atomic<int> cancel{0};
    uint32_t ordinal = 0;            // the job's place among the context's submissions, from 1: the same on every rank
    bool started = false;            // the worker has taken the job (a multi-GPU cancel then writes the stop board), under `mu`
    PinnedBlock result_block;
    tad_rows rows{};
    double t_submit = 0;
    uint32_t passes = 0;             // hash-range passes the job ran in (tad_job_memory)
    tad_progress prog{};             // passes and ARIMA fits so far (tad_job_progress), under `mu`
    uint64_t peak_workspace = 0;     // largest device workspace the context held while the job ran
    // fit sharing (tad_set_fit_sharing)
    uint64_t share = 0;              // an ARIMA job whose fit yields: the reserve read when it started (0: it does not)
    bool no_interleave = false;      // did not fit a reserve: waits for its turn in the queue
    uint32_t yields = 0;             // times the fit phase yielded (tad_job_yields), under `mu`
    double parked_ms = 0;            // time the job was parked, under `mu`
    double quiet_until = 0;          // now_ms() before which the fit does not yield again
    // lending (TAD_FLAG_LEND): a streamed job runs queued jobs while it waits for its caller (lend)
    uint64_t lend = 0;               // the reserve read when it started (0: it does not lend)
    uint32_t lent_jobs = 0;          // jobs run in its lends (tad_job_lent), under `mu`
    double lent_ms = 0;              // time it was lent, under `mu`
    double lend_until = 0;           // now_ms() before which it does not lend again
    // streamed input (tad_submit_stream): the caller hands the worker one column block at a time, under `mu`.  `cols`
    // then holds the first block: its non-NULL columns are the set every block must carry.
    bool stream = false;
    bool rank_stream = false;        // this rank's part of a job streamed to every rank (TAD_FLAG_RANK_STREAM)
    std::atomic<int> peer_stop{0};   // a rank stream job: a peer's stop for it was read off this rank's board
    uint64_t rows_hint = 0;          // the caller's estimate of one round's rows (0 = unknown)
    uint64_t round_rows = 0;         // rows of the first round (tad_status.rows_in)
    uint64_t stored_rows = 0;        // rows the host row store held for the passes (tad_job_host_memory)
    uint64_t peak_host = 0;          // most store bytes the context held while the job ran
    struct {
        tad_columns blk{};           // handed over, not yet taken by the worker
        bool has_blk = false;
        bool end_req = false;        // the caller closed the round; cleared when the worker finishes with it
        bool round_done = false;     // the worker finished with the round; `again` is valid
        bool again = false;
        bool input_done = false;     // tad_stream_end returned again = 0
        tad_text_column txt[4]{};    // the handed-over block's text slots (tad_stream_push_text_ns)
        uint64_t pushed = 0, taken = 0, released = 0;   // blocks handed over / taken / no longer read by the engine
        uint64_t round_start = 0;    // `taken` when the last round was closed
        int err = 0;                 // a bad block: the worker fails the job with this code and message
        char msg[200] = {0};
    } in;
    // text slots (tad_stream_push_text_ns), set by the first block: src_ip / dst_ip arrive as Native String bytes and
    // are dictionary-encoded on the device; src_ns / dst_ns (slots 2, 3) are only tested against the ignore list's
    // names.  On completion each key slot's dictionary is copied here (tad_job_names).
    bool text[4] = {false, false, false, false};
    std::vector<uint8_t> names[2];
    std::vector<uint64_t> names_off[2];
    // row predicates (tad_submit_stream_filtered): per text slot a TAD_NAME_* op and its pattern, and proto_eq (-1: none)
    int32_t name_op[2] = {TAD_NAME_ANY, TAD_NAME_ANY};
    std::vector<uint8_t> name_pat[2];
    int32_t proto_eq = -1;
    // the ignore list as names (tad_submit_stream_filtered_ns): its device image (ns_list_image) and name count; the
    // row filter's list `ns_ignore` is then {kNsListed}, the verdict the namespace slots stage per row
    std::vector<uint8_t> ns_image;
    uint32_t ns_names = 0;
    bool filtered() const { return name_op[0] != TAD_NAME_ANY || name_op[1] != TAD_NAME_ANY || proto_eq >= 0; }
};

struct tad_ctx {
    tad_config cfg{};
    cudaStream_t stream = nullptr, copy_stream = nullptr;
    cudaEvent_t ev[kMaxEvents]{};
    cudaEvent_t ev_alt[2][kMaxEvents]{};  // ev of the jobs run while an ARIMA pass is parked, one set per level of parking
                                          // (a fit beside a parked one can yield too): each parked pass keeps its times
    int park_depth = 0;                   // ARIMA passes parked now (Parked)
    YieldedFit *beside = nullptr;         // while a fit's yield runs jobs: the fit a flagged ARIMA job may fit beside
    cudaEvent_t chunk_ev[kMaxChunks]{};
    cudaEvent_t start_ev = nullptr;
    cudaEvent_t x_ev[kMaxXChunks + 1]{};
    int exchange_chunks = kMaxXChunks;
    bool exchange_chunks_forced = false;     // TAD_EXCHANGE_CHUNKS given: use it at every world size
    uint64_t exchange_min_rows = 1u << 22;   // below this the exchange is not worth chunking (TAD_EXCHANGE_MIN_ROWS)
    std::mutex mu;
    std::condition_variable cv;
    std::deque<tad_job *> queue;
    std::thread worker;
    bool stop = false;
    std::atomic<int> stopping{0};                   // tad_shutdown: a streamed job waiting for input is cancelled
    int debug_logb = -1;
    bool debug_no_grow = false;  // TAD_DEBUG_NO_GROW=1: a first streamed round's guarded pass columns never grow (RoundGrowth),
                                 // so that the tests reach its count-only fallback
    uint64_t text_mask = ~0ull;  // TAD_DEBUG_TEXT_MASK (hex): ANDed into the name hashes of the text dictionaries and the
                                 // ignore list, so that the tests can make names collide
    int debug_target = 0;      // TAD_GROUP_TARGET: mean rows per bucket (tuning)
    int num_sms = 132;
    // device workspace (grow-only, reused across jobs; jobs are serialized by the worker)
    DevBuf d_col[10], hist, offsets, cursor, big_list, big_base, cls_list, csr_p, stats, part, csr_v, csr_t, nsb, npb, sbase, outb, ns_ignore, spill,
        dbx, dbi, exch, scan_sync, small, hist_all, seg_off, seg_total, entries, ar_y, ar_pred, ar_lam, ar_res, ovf;
    int optimistic = 1;      // TAD_OPTIMISTIC=0: always the exact (histogram + scan + scatter) partition
    unsigned long long *h_small = nullptr;   // pinned, kSmallWords x u64
    // Word offsets in h_small and in the device scratch `small` (d_small) that mirrors it.  From word 0: gather_small, the
    // exact partition's rows per segment, the pass counts.  The regions one path uses together do not overlap.
    static constexpr int kSmallWords = 256, kSmallDevWords = 512, kGatherMax = 16;   // kGatherMax: largest gather_small message
    static constexpr int kWOvf = 32;          // multi-GPU slot path: every rank's overflow rows
    static constexpr int kWPullSkip = 40;     // exact pull: rows in front of my bucket range in every rank's partition
    static constexpr int kWBarrier = 48, kWBarrierIn = 56;   // peer barrier (d_small only): the word sent, the words received
    static constexpr int kWSendLo = 64;       // NCCL exchange: send boundaries of every chunk, kMaxRanks + 1 per chunk
    static constexpr int kWPassCursor = 128;  // hash-range passes: the pass cursor alone, read while the counts are held
    static constexpr int kWTextState = 192;   // text slots: 8 state words per dictionary, then the ignore list's 16
    static_assert(kGatherMax * (1 + kMaxRanks) <= kSmallWords && kSmallWords <= kSmallDevWords, "small scratch size");
    static_assert(kMaxSeg <= kWOvf && kWOvf + kMaxRanks <= kWPullSkip && kWPullSkip + kMaxRanks <= kWBarrier &&
                  kWBarrier < kWBarrierIn && kWBarrierIn + kMaxRanks <= kWSendLo &&
                  kWSendLo + kMaxXChunks * (kMaxRanks + 1) <= kSmallWords, "partition scratch regions overlap");
    static_assert(kMaxPasses + 1 <= kWPassCursor && kWPassCursor < kWTextState && kWTextState + 4 * 8 <= kSmallWords,
                  "pass scratch regions overlap");
    uint32_t scan_epoch = 0;
    uint32_t *h_stats = nullptr;   // pinned readback of the device scalars
    // Pinned words of the fit launch in flight (wait_fit).  Per part ([0] the job's own fit, [1] the yielded fit beside
    // it): its counters (fits_total, fits_done) as last copied back while the kernel runs and once it has ended, and its
    // redo words (the fits its leave dropped; of those, finished again).  Then the values a cancel (1) and a leave (2)
    // copy into a cancel word, and the yielded fit's lowest unfinished series (launch_arima_unfinished).
    struct FitCounts { uint32_t total, done; };
    struct FitWords { FitCounts run, end; uint32_t dropped, redone; };
    struct FitPinned { FitWords part[2]; uint32_t cancel = 1, leave = 2, from = 0; };
    FitPinned *h_fit = nullptr;
    std::atomic<uint64_t> fit_share{0};             // tad_set_fit_sharing: the reserve of the jobs run beside a fit (0: off)
    cudaEvent_t fit_ev[2]{};        // [0]: the fit counters are reset; [1]: the fit kernel has ended
    cudaEvent_t fits_ev = nullptr;  // a copy of the fit counters has reached h_fit
    std::mutex pool_mu;
    std::vector<PinnedBlock> pinned_pool;
    NcclComm nccl;
    NumaInfo numa;                                  // NUMA node of the GPU: pinned buffers and the worker thread live there
    // multi-GPU optimistic partition + peer pull (DESIGN.md section 6): every rank scatters into fixed-capacity slots of an
    // exported buffer (arrival counters in front, slots behind), the peers map it (CUDA IPC) and the owner's group kernel
    // pulls its bucket segments over NVLink -- no histogram pass, no all-to-all, no receive buffer.
    int peer_pull = 1;                              // TAD_PEER_PULL=0: always the exact partition + NCCL all-to-all
    int sort_classes = 0;                           // TAD_SORT_CLASSES=1: capacity-class bucket lists sorted by bucket before the group phase
    DevBuf sortb;
    int exact_pull = 0;                             // TAD_EXACT_PULL=1: the exact partition is pulled by the peers too (no receive buffer)
    size_t x_budget = 32ull << 30;                  // largest exported slot buffer (TAD_SLOT_BUDGET_GB; 40 % of an 80 GB H100); beyond it: exact partition
    DevBuf xbuf;                                    // exported: [counters: B x u32, padded][slots: B x slot x Row32]
    void *peer_x[kMaxRanks]{};                      // peers' xbuf mapped into this process
    bool peers_mapped = false;
    // stop board of a multi-GPU context (DESIGN.md section 6): kMaxRanks u32 in device memory, word r the ordinal of the
    // last job rank r cancelled (0: none), read by the fit kernel every round.  Each rank writes its own word into every
    // board it has mapped (post_stop); a word has one writer and only grows.
    uint32_t job_seq = 0;                           // ordinals of the jobs queued so far, under `mu`
    uint32_t *board = nullptr;
    uint32_t *peer_board[kMaxRanks]{};              // rank r's board as mapped here ([rank] = board); null: not mapped
    bool boards_shared = false;                     // the ranks have exchanged their boards' handles (the same on every rank)
    std::mutex board_mu;                            // post_stop
    cudaStream_t board_stream = nullptr;            // non-blocking: a board write waits for no job's work
    uint32_t *h_board = nullptr;                    // pinned: [0] the ordinal this rank last wrote; [8, 16) its board read back
    size_t x_agreed = 0;                            // exported size all ranks agreed on at the last (re)mapping
    DevBuf xcnt, xtotal;                            // per-source counts / totals of the owned bucket range
    // memory budget and hash-range passes (DESIGN.md section 9)
    std::atomic<uint64_t> budget{0};                // tad_set_memory_budget; 0 = free device memory at job start + held - headroom
    size_t held = 0;                                // device bytes the workspace holds (ensure)
    size_t peak = 0;                                // largest `held` since the running job started
    size_t limit = 0;                               // while a job runs under a budget: ensure() never grows `held` past it
    DevBuf stage, pcnt;                             // pass mode: double-buffered host chunk staging; pass counters + cursor
    cudaEvent_t stage_ev[2]{};                      // staging half free again (the split kernel of its last chunk is done)
    cudaEvent_t blk_ev[2]{};                        // streamed input: the engine has finished reading a caller's block
    // host row store (DESIGN.md section 11): pinned pages that keep a streamed round's rows for the job's passes
    std::atomic<uint64_t> host_budget{0};           // tad_set_host_budget; 0 = no store
    std::vector<PinnedBlock> store_slabs;           // pinned slabs of up to 64 MiB, carved into pages
    std::vector<char *> store_free;                 // pages holding no job's rows
    size_t store_page = 0;                          // page bytes
    size_t store_held = 0, store_peak = 0;          // pinned bytes of the slabs; their most since the running job started
    DevBuf ostage;                                  // out-stage: two halves of packed rows, count matrix, scan scratch, chunk counts
    cudaStream_t d2h_stream = nullptr;              // copies from the out-stage to the store
    cudaEvent_t ost_ev[2]{};                        // out-stage half free again (its copies to the store are done)
    cudaEvent_t cnt_ev[2]{};                        // a chunk's residue counts have reached h_chunk
    uint32_t *h_chunk = nullptr;                    // pinned, 2 x 64: rows per residue of the last two chunks
    // text key slots (DESIGN.md section 10, "Text keys on the device"): one dictionary per slot, alive for one job
    struct TextSlot {
        DevBuf slots, minrow, slot_id, arena, off, hash, state;
        DevBuf keep, pat;                           // a filtered job: the predicate's byte per name; its pattern
        uint32_t cap = 0;                           // table slots (0: no dictionary yet)
        uint64_t names_ub = 0, bytes_ub = 0;        // upper bounds of its names / arena bytes, exact after each readback
        std::vector<DevBuf *> bufs() { return {&slots, &minrow, &slot_id, &arena, &off, &hash, &state, &keep, &pat}; }
        void swap_sizes(TextSlot &o)                // a parked slot's sizes are parked with its buffers
        {
            std::swap(cap, o.cap);
            std::swap(names_ub, o.names_ub);
            std::swap(bytes_ub, o.bytes_ub);
        }
    } tdict[2];
    DevBuf tstage, tscratch;                        // a chunk's marks and text bytes; the encode scratch
    DevBuf nsl;                                     // the ignore list of namespace text slots (ns_list_image)
};

namespace {

const char *kErrNames[] = {"ok", "invalid argument", "CUDA error", "out of memory", "NCCL error", "illegal state",
                           "cancelled", "unsupported", "internal error"};

struct JobFail {
    int code;
    char msg[256];
};

[[noreturn]] void fail(int code, const char *fmt, ...)
{
    JobFail f;
    f.code = code;
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(f.msg, sizeof(f.msg), fmt, ap);
    va_end(ap);
    throw f;
}

#define CU(expr)                                                                                         \
    do {                                                                                                 \
        cudaError_t _e = (expr);                                                                         \
        if (_e != cudaSuccess)                                                                           \
            fail(_e == cudaErrorMemoryAllocation ? TAD_ERR_NOMEM : TAD_ERR_CUDA, "%s: %s (%s:%d)", #expr, \
                 cudaGetErrorString(_e), __FILE__, __LINE__);                                            \
    } while (0)

size_t alloc_bytes(size_t bytes) { return (bytes + bytes / 16 + 256 + 255) & ~size_t(255); }   // what ensure() asks for
size_t exact_bytes(size_t bytes) { return (bytes + 255) & ~size_t(255); }

// Whether the workspace may grow by `extra` bytes inside the budget (always, without one).
bool can_grow(const tad_ctx *ctx, size_t extra) { return !ctx->limit || ctx->held + extra <= ctx->limit; }

// Whether ensure(b, bytes) stays inside the budget.
bool fits(const tad_ctx *ctx, const DevBuf &b, size_t bytes)
{
    return bytes <= b.cap || can_grow(ctx, exact_bytes(bytes) - b.cap);
}

// The allocate step: a new block of at least `bytes`, counted in `held` and `peak`.  Under a budget (ctx->limit != 0) the
// 1/16 slack is dropped where it would not fit, and growth past the budget is a planning error: the planner sized every
// buffer it can know in advance.  A failed cudaMalloc is retried once at the exact size.
DevBuf alloc_buf(tad_ctx *ctx, size_t bytes)
{
    size_t want = alloc_bytes(bytes);
    if (!can_grow(ctx, want)) want = exact_bytes(bytes);
    if (!can_grow(ctx, want))
        fail(TAD_ERR_INTERNAL, "workspace would grow to %zu bytes, past the memory budget of %zu bytes", ctx->held + want, ctx->limit);
    DevBuf b;
    if (cudaMalloc(&b.p, want) != cudaSuccess) {
        cudaGetLastError();
        want = exact_bytes(bytes);
        CU(cudaMalloc(&b.p, want));
    }
    b.cap = want;
    ctx->held += want;
    ctx->peak = std::max(ctx->peak, ctx->held);
    return b;
}

// The free step: `b` is freed and empty, and `held` leaves it out.  Returns the cudaFree's error, for the callers that
// free on a context with a sticky error (a failed job's cleanup) and go on.
cudaError_t drop_buf(tad_ctx *ctx, DevBuf &b)
{
    const cudaError_t e = b.p ? cudaFree(b.p) : cudaSuccess;
    ctx->held -= b.cap;
    b = DevBuf{};
    return e;
}

void free_buf(tad_ctx *ctx, DevBuf &b) { CU(drop_buf(ctx, b)); }

// Grow-only workspace buffer (freed before it is allocated again).
void ensure(tad_ctx *ctx, DevBuf &b, size_t bytes)
{
    if (bytes <= b.cap) return;
    free_buf(ctx, b);
    b = alloc_buf(ctx, bytes);
}

// A pass whose oversized-bucket spill scratch or result buffer (sizes known only while it runs) would not fit the budget:
// the job driver splits it by the next hash bit.  `what` needed `bytes` beside the `held` bytes of workspace.
struct PassSplit {
    const char *what = "";
    size_t bytes = 0, held = 0;
};

// Lifetimes of the workspace buffers (workspace_bufs).  kJobs and kPasses name the events a buffer is kept across (the
// others free it); kParked, what a parked ARIMA pass, or a streamed job lending the GPU, takes out of the context.
constexpr int kJobs = 1;     // kept when a job ends: all but the text key dictionaries, which live for one job
constexpr int kPasses = 2;   // kept across the passes of a job: what every pass reads (free_pass_buffers frees the rest)
constexpr int kParked = 4;   // moved out of the context while a pass is parked (Parked), the rest left for reuse
constexpr uint64_t kBudgetFloor = 64ull << 20;     // smallest memory budget tad_set_memory_budget accepts

// Every workspace buffer with its lifetime, the exported multi-GPU buffer `xbuf` apart (ranks agree on its size).
//
// Kept across passes: the pass columns d_col[0..8), the staging, the pass counters, the stats words, the ns_ignore list
// (ids, and the names of namespace text slots), the text key dictionaries and their staging, and `small` (run_pipeline
// ensures it first anyway).
//
// Parked: a parked ARIMA pass moves out the buffers the rest of its fit, its detect_arima and its pass driver read
// (ctx->held leaves them out).  Everything else stays for the jobs run meanwhile to reuse: each plans under the reserve
// and frees the workspace first when it does not fit there (run_job), so the parked bytes plus theirs stay inside the
// budget the ARIMA job planned in plus the reserve.  Nothing is freed before they run, which would sit in their wait
// (cudaFree); their workspace is freed at the restore, after they have completed.  The parked buffers:
//   the fit and detect_arima: the series entries (`entries` after the optimistic partition, in place in `part` after the
//     exact one), offsets, sbase, csr_v, csr_t, ar_y, ar_pred, ar_lam, the resume points ar_res, the stats words (fit
//     counters, cancel word, result count) and outb, into which the pass's result layout points;
//   the pass driver (run_passes), which took pointers to them at its start: the pass columns d_col[0..8), the staging,
//     the pass counters and the ns_ignore list;
//   a streamed job's text key slots: both dictionaries (table, arena, offsets, hashes, keep bytes, pattern, state words,
//     with their sizes), which its later rounds look names up in and its end copies out, so its ids stay the same, and
//     the text staging and encode scratch its sweeps take as sized, and the ignore list its namespace text slots are
//     tested against in every later round.  They were planned in the budget less the reserve.
// A streamed job lending the GPU (lend) parks between two blocks of a round, or before its first block, with these same
// buffers.  Besides them its sweep reads, between two blocks, the pass counters and cursor (pcnt), the pass columns, the
// double-buffered staging (a host row store round may have a partly filled half), the open dictionaries with their
// sizes, the namespace list image and the out-stage of a round going to the host row store (ostage, two halves of
// packed rows whose copies to the pages are issued with the next chunk): all parked.  Its planning state and sweep
// cursors are host variables of run_passes, and the events it waits for between blocks (stage_ev, blk_ev, ost_ev,
// cnt_ev) have completed before the lend (its streams are synchronised) and are either left alone by the lent jobs or
// recorded by them on work that has ended before the restore.  A fit's pass never holds the out-stage: a round frees it
// at its end (RowStore::end).
// What else a parked streamed pass needs is not in the workspace and no interleaved job touches it: the job's stream
// input state (tad_job::in: its feeder, blocked in a push or end call, goes on with the same round) and the host row
// store pages of its passes (its RowStore's lists and pinned chunk counts h_chunk, which only a streamed round uses; a
// lend runs no streamed job).  An interleaved job takes store pages only from the free list and new slabs within the
// host budget less the slabs held (store_share), and frees no slab.
// What the interleaved jobs may overwrite is rebuilt before the ARIMA job reads it again:
//   hist, cursor, big_list, big_base, cls_list, nsb, npb, csr_p, ovf, spill, sortb, dbx, dbi, small: the partition and
//     group scratch, which the next pass's pipeline ensures and writes before reading (scan_sync: freed at the restore, so
//     that pipeline allocates and zeroes it again for the scan's epochs);
//   d_col[8..10): a one-pass job's host namespace columns, read before the fit only;
//   h_stats and h_small: read back again after the fit (read_stats) and after every sweep (the counts);
//   h_fit: the fit counters are published before the park;
//   ev: the interleaved jobs record ev_alt, so the pass's phase events survive; the other events of a sweep are
//     recorded in that sweep before they are waited for;
//   limit, peak and store_peak: restored.
std::vector<std::pair<DevBuf *, int>> workspace_bufs(tad_ctx *ctx)
{
    tad_ctx &c = *ctx;
    std::vector<std::pair<DevBuf *, int>> v;
    auto add = [&](int life, const std::vector<DevBuf *> &bufs) {
        for (DevBuf *b : bufs) v.push_back({b, life});
    };
    add(kJobs, {&c.hist, &c.cursor, &c.big_list, &c.big_base, &c.cls_list, &c.csr_p, &c.nsb, &c.npb, &c.ovf, &c.spill,
                &c.sortb, &c.dbx, &c.dbi, &c.scan_sync, &c.exch, &c.hist_all, &c.seg_off, &c.seg_total, &c.xcnt,
                &c.xtotal, &c.d_col[8], &c.d_col[9]});
    add(kJobs | kPasses, {&c.small});
    add(kJobs | kParked, {&c.part, &c.entries, &c.offsets, &c.sbase, &c.csr_v, &c.csr_t, &c.ar_y, &c.ar_pred, &c.ar_lam,
                          &c.ar_res, &c.outb, &c.ostage});
    add(kJobs | kPasses | kParked, {&c.stats, &c.stage, &c.pcnt, &c.ns_ignore, &c.tstage, &c.tscratch, &c.nsl});
    for (int i = 0; i < 8; i++) add(kJobs | kPasses | kParked, {&c.d_col[i]});
    for (auto &t : c.tdict) add(kPasses | kParked, t.bufs());
    return v;
}

// The free step over the list: every workspace buffer whose lifetime has no flag of `keep` is freed, also on a context
// with a sticky error; returns the first error.  A text key slot without buffers has no dictionary: its sizes go too.
cudaError_t free_bufs(tad_ctx *ctx, int keep = 0)
{
    cudaError_t e = cudaSuccess;
    for (auto [b, life] : workspace_bufs(ctx)) {
        const cudaError_t f = (life & keep) ? cudaSuccess : drop_buf(ctx, *b);
        if (e == cudaSuccess) e = f;
    }
    for (auto &t : ctx->tdict)
        if (!t.state.p) {
            t.cap = 0;
            t.names_ub = t.bytes_ub = 0;
        }
    return e;
}

void free_workspace(tad_ctx *ctx) { CU(free_bufs(ctx)); }

PinnedBlock take_pinned(tad_ctx *ctx, size_t bytes)
{
    {
        std::lock_guard<std::mutex> lk(ctx->pool_mu);
        int best = -1;
        for (size_t i = 0; i < ctx->pinned_pool.size(); i++)
            if (ctx->pinned_pool[i].cap >= bytes && (best < 0 || ctx->pinned_pool[i].cap < ctx->pinned_pool[best].cap))
                best = (int)i;
        if (best >= 0) {
            PinnedBlock b = ctx->pinned_pool[best];
            ctx->pinned_pool.erase(ctx->pinned_pool.begin() + best);
            return b;
        }
    }
    PinnedBlock b;
    b.cap = (bytes + bytes / 8 + 4095) & ~size_t(4095);
    NumaScope numa(ctx->numa);
    CU(cudaHostAlloc(&b.p, b.cap, cudaHostAllocDefault));
    return b;
}

void give_pinned(tad_ctx *ctx, PinnedBlock b)
{
    if (!b.p) return;
    std::lock_guard<std::mutex> lk(ctx->pool_mu);
    ctx->pinned_pool.push_back(b);
}

// ---- host row store pages (worker thread only) ------------------------------------------------------------------------
constexpr uint64_t kStoreSlab = 64ull << 20;

// budget / 1024 rounded to a MiB, within [1, 64] MiB: the 64 partly filled pages (one per residue) waste at most 1/16
size_t store_page_bytes(uint64_t budget)
{
    const uint64_t mib = (budget / 1024 + (1u << 19)) >> 20;
    return (size_t)std::min<uint64_t>(64, std::max<uint64_t>(1, mib)) << 20;
}

// Before a job: the slabs above the budget are freed (all of them when the page size changes) and every page is free.
// Returns the budget it read: the job's host budget, so that the page size and the budget the job fills stay one pair
// whatever tad_set_host_budget does while the job runs.
uint64_t store_trim(tad_ctx *ctx)
{
    const uint64_t budget = ctx->host_budget.load();
    const size_t page = budget ? store_page_bytes(budget) : 0;
    while (!ctx->store_slabs.empty() && (page != ctx->store_page || ctx->store_held > budget)) {
        cudaFreeHost(ctx->store_slabs.back().p);
        ctx->store_held -= ctx->store_slabs.back().cap;
        ctx->store_slabs.pop_back();
    }
    ctx->store_page = page;
    ctx->store_free.clear();
    for (const PinnedBlock &s : ctx->store_slabs)
        for (size_t o = 0; o + page <= s.cap; o += page) ctx->store_free.push_back(static_cast<char *>(s.p) + o);
    ctx->store_peak = ctx->store_held;
    return budget;
}

// store_trim for a job run while an ARIMA pass is parked (interleave): the parked job's pages stay where they are, so no
// slab is freed and the free list is kept.  The job takes free pages and new slabs within the host budget less every slab
// held, the parked job's included.  Returns the budget it read, or 0 (no store) when its page size is not the context's.
uint64_t store_share(tad_ctx *ctx)
{
    const uint64_t budget = ctx->host_budget.load();
    const size_t page = budget ? store_page_bytes(budget) : 0;
    if (!page || (ctx->store_page && page != ctx->store_page)) return 0;
    ctx->store_page = page;          // was 0: the context holds no slab
    ctx->store_peak = ctx->store_held;
    return budget;
}

// A free page; a new slab when none is left.  Null when the slab would pass the budget or cannot be pinned.
char *store_take_page(tad_ctx *ctx, uint64_t budget)
{
    if (ctx->store_free.empty()) {
        const size_t page = ctx->store_page;
        const uint64_t room = budget > ctx->store_held ? budget - ctx->store_held : 0;
        const size_t n = (size_t)std::min<uint64_t>(kStoreSlab / page, room / page);
        if (n == 0) return nullptr;
        PinnedBlock s;
        s.cap = n * page;
        NumaScope numa(ctx->numa);
        if (cudaHostAlloc(&s.p, s.cap, cudaHostAllocDefault) != cudaSuccess) {
            cudaGetLastError();
            return nullptr;
        }
        ctx->store_slabs.push_back(s);
        ctx->store_held += s.cap;
        ctx->store_peak = std::max(ctx->store_peak, ctx->store_held);
        for (size_t o = 0; o < s.cap; o += page) ctx->store_free.push_back(static_cast<char *>(s.p) + o);
    }
    char *p = ctx->store_free.back();
    ctx->store_free.pop_back();
    return p;
}

void set_progress(tad_job *job, int state, int completed)
{
    std::lock_guard<std::mutex> lk(job->mu);
    job->st.state = state;
    job->st.completed_stages = std::max(job->st.completed_stages, completed);    // passes rerun the stages
}

tad_progress progress_of(tad_job *job)
{
    std::lock_guard<std::mutex> lk(job->mu);
    return job->prog;
}

// tad_job_progress's pass counts.  fits_before: the job's counts before a pass that has just been split, which gives its
// fits back (its halves fit the same series again); null: the fit counts stay.
void set_passes(tad_job *job, uint32_t done, uint32_t planned, const tad_progress *fits_before = nullptr)
{
    std::lock_guard<std::mutex> lk(job->mu);
    job->prog.passes_done = done;
    job->prog.passes = planned;
    if (fits_before) {
        job->prog.fits_done = fits_before->fits_done;
        job->prog.fits_total = fits_before->fits_total;
    }
}

bool run_one(tad_ctx *ctx, tad_job *job, uint64_t reserve);
void release_blocks(tad_job *job, uint64_t n);

// Whether a fit's yield may hand its place to `j`, a queued job: an EWMA or DBSCAN job that has not been found too
// large for the reserve.  A streamed one only with TAD_FLAG_SHARE and once its feeder has handed over its first block or
// closed its round: a job whose caller has not started delivering would hold the fit parked while it waits.
// `beside`: the yield is that of a fit parked at the outer level whose reserve halves to the 64 MiB floor or more; then an
// ARIMA job with TAD_FLAG_FIT_BESIDE may run too, and fits beside it (fit_beside): a tad_submit one, or a streamed one
// with TAD_FLAG_SHARE as well, fed as above.
// `lend`: the hand-over is a streamed job's lend, which runs tad_submit EWMA and DBSCAN jobs only: an ARIMA fit would keep
// its caller waiting for minutes, and a streamed job's own caller could leave the GPU idle in turn.
bool interleavable(tad_job *j, bool beside, bool lend = false)
{
    if (j->no_interleave) return false;
    if (lend) return !j->stream && (j->spec.algo == TAD_ALGO_EWMA || j->spec.algo == TAD_ALGO_DBSCAN);
    if (j->spec.algo == TAD_ALGO_ARIMA) {
        if (!beside || !(j->spec.flags & TAD_FLAG_FIT_BESIDE)) return false;
    } else if (j->spec.algo != TAD_ALGO_EWMA && j->spec.algo != TAD_ALGO_DBSCAN) {
        return false;
    }
    if (!j->stream) return true;
    if (!(j->spec.flags & TAD_FLAG_SHARE)) return false;
    std::lock_guard<std::mutex> lk(j->mu);
    return j->in.pushed > 0 || j->in.end_req;
}

// Whether a yield of `job`'s fit may run an ARIMA job beside it: the job parks at the outer level (a job fitting beside a
// parked fit takes no ARIMA partner) and half its reserve, the partner's budget, is at least the 64 MiB floor.
bool beside_ok(const tad_ctx *ctx, const tad_job *job)
{
    return ctx->park_depth == 0 && job->share / 2 >= kBudgetFloor;
}

// Whether a yield (a lend) would run a job now: a cancelled one is not worth it (it fails at once in its turn).
bool interleave_waiting(tad_ctx *ctx, const tad_job *job, bool lend = false)
{
    const bool beside = !lend && beside_ok(ctx, job);
    std::lock_guard<std::mutex> lk(ctx->mu);
    for (tad_job *j : ctx->queue)
        if (interleavable(j, beside, lend) && !j->cancel.load()) return true;
    return false;
}

// A lending job's caller has handed over a block or closed its round: the lend ends before the next queued job.
bool input_ready(tad_job *job)
{
    std::lock_guard<std::mutex> lk(job->mu);
    return job->in.has_blk || job->in.end_req;
}

// A parked ARIMA pass: the buffers workspace_bufs() marks kParked, with the dictionaries' sizes, are moved out of the
// context into `bufs` and `dict`, and ctx->held leaves them out.
struct Parked {
    tad_ctx *ctx;
    std::vector<std::pair<DevBuf *, DevBuf>> bufs;
    tad_ctx::TextSlot dict[2];       // the dictionaries' sizes (their buffers are in `bufs`)
    size_t limit, peak, store_peak;
    bool out = false;

    Parked(tad_ctx *c) : ctx(c), limit(c->limit), peak(c->peak), store_peak(c->store_peak)
    {
        CU(cudaStreamSynchronize(ctx->stream));
        CU(cudaStreamSynchronize(ctx->copy_stream));
        for (auto [b, life] : workspace_bufs(ctx)) {
            if (!(life & kParked) || !b->p) continue;
            bufs.push_back({b, *b});
            ctx->held -= b->cap;
            *b = DevBuf{};
        }
        for (int t = 0; t < 2; t++) ctx->tdict[t].swap_sizes(dict[t]);
        out = true;
        std::swap(ctx->ev, ctx->ev_alt[ctx->park_depth++]);
    }
    // the interleaved jobs' workspace is freed and the parked buffers return; drop: they are freed too (a cancel)
    void restore(bool drop = false)
    {
        if (!out) return;
        out = false;
        std::swap(ctx->ev, ctx->ev_alt[--ctx->park_depth]);
        cudaStreamSynchronize(ctx->stream);
        cudaStreamSynchronize(ctx->copy_stream);
        free_bufs(ctx);
        for (auto [b, parked] : bufs) {
            *b = parked;
            ctx->held += parked.cap;
        }
        bufs.clear();
        for (int t = 0; t < 2; t++) ctx->tdict[t].swap_sizes(dict[t]);
        if (drop) free_bufs(ctx);
        ctx->limit = limit;
        ctx->peak = std::max(peak, ctx->held);
        ctx->store_peak = store_peak;
    }
    ~Parked() { restore(); }
};

// Runs the eligible jobs queued now, in FIFO order, while the ARIMA pass of `job` is parked: each inside the reserve
// (run_one), so one whose 1/64 hash range does not fit it is put back where it was and runs in its turn.  A cancel of
// `job` takes effect once the job in progress has ended: the parked buffers are freed and the job fails.
// At most one ARIMA job (TAD_FLAG_FIT_BESIDE) runs per yield, the first queued: its fit runs beside the rest of `job`'s,
// described by `yf` (ctx->beside while the batch runs).
// `lend`: `job` is a streamed job lending the GPU while it waits for its caller (lend): the jobs run in its lend reserve,
// and the batch also stops once its caller hands over a block or closes its round, so a pushed block waits for at most
// one job.  Returns the number of jobs run (those put back left out).
uint32_t interleave(tad_ctx *ctx, tad_job *job, YieldedFit *yf, bool lend = false)
{
    std::vector<tad_job *> batch;
    bool beside = yf && beside_ok(ctx, job);
    {
        std::lock_guard<std::mutex> lk(ctx->mu);
        for (tad_job *j : ctx->queue)
            if (interleavable(j, beside, lend)) {
                batch.push_back(j);
                if (j->spec.algo == TAD_ALGO_ARIMA) beside = false;
            }
    }
    const double t0 = now_ms();
    Parked park(ctx);
    if (yf && ctx->park_depth == 1) ctx->beside = yf;
    const double t1 = now_ms();
    uint32_t ran = 0;
    for (tad_job *j : batch) {
        if (job->cancel.load() || (lend && input_ready(job))) break;
        size_t at;
        {
            std::lock_guard<std::mutex> lk(ctx->mu);       // only this thread takes jobs out of the queue
            at = (size_t)(std::find(ctx->queue.begin(), ctx->queue.end(), j) - ctx->queue.begin());
            if (at == ctx->queue.size()) continue;
            ctx->queue.erase(ctx->queue.begin() + at);
        }
        if (run_one(ctx, j, lend ? job->lend : job->share)) {
            ran++;
        } else {
            std::lock_guard<std::mutex> lk(ctx->mu);       // jobs submitted meanwhile went behind it
            ctx->queue.insert(ctx->queue.begin() + at, j);
        }
    }
    if (ctx->beside == yf) ctx->beside = nullptr;
    CU(cudaSetDevice(ctx->cfg.device));
    const double t2 = now_ms();
    const bool cancelled = job->cancel.load() != 0;
    park.restore(cancelled);
    if (getenv("TAD_DEBUG_YIELD"))
        fprintf(stderr, "%s: park %.2f ms, %u of %zu jobs %.2f ms, restore %.2f ms\n", lend ? "lend" : "yield", t1 - t0,
                ran, batch.size(), t2 - t1, now_ms() - t2);
    if (cancelled) fail(TAD_ERR_CANCELLED, "job cancelled");
    return ran;
}

// ---- lending the GPU while a streamed job waits for its caller (TAD_FLAG_LEND) --------------------------------------------
// A streamed job's worker waits in next_block until its caller hands over the next block or closes the round; the
// caller's source (a ClickHouse SELECT) is usually far slower than the GPU.  A job with TAD_FLAG_LEND started while fit
// sharing was on (job->lend: the reserve) runs the queued tad_submit EWMA and DBSCAN jobs meanwhile (interleave), its
// workspace parked as a yielded fit's is (workspace_bufs), and resumes once a block is pending or the round has ended.
//
// kLendWaitMs: how long the worker must have waited in one next_block call before it lends.  A caller that pushes
// back to back hands the next block over within the first poll of the wait loop (5 ms), so a lend there would only make
// that block wait for a job; a caller whose source has stalled for longer is slower than any lent job's parking
// overhead.  DESIGN.md section 10 ("Lending the GPU while a streamed job waits") has the measurement.
constexpr double kLendWaitMs = 5.0;

// Called by next_block, without the job's lock, once the worker has waited `waited` ms in it: lends when every rule
// holds.  Before lending the context's streams are synchronised, so that every block taken has been read, and those
// blocks are released: no push waits for a lend it does not need to.  Fairness as for a fit's yields: after a lend the
// job does not lend again until as much time has passed as the lend took.
void lend(tad_job *job, double waited)
{
    tad_ctx *ctx = job->ctx;
    if (!job->lend || ctx->park_depth > 0 || waited < kLendWaitMs || now_ms() < job->lend_until ||
        !interleave_waiting(ctx, job, true))
        return;
    CU(cudaStreamSynchronize(ctx->stream));
    CU(cudaStreamSynchronize(ctx->copy_stream));
    CU(cudaStreamSynchronize(ctx->d2h_stream));
    uint64_t taken;
    {
        std::lock_guard<std::mutex> lk(job->mu);
        taken = job->in.taken;
    }
    release_blocks(job, taken);
    const double t0 = now_ms();
    const uint32_t ran = interleave(ctx, job, nullptr, true);
    const double t1 = now_ms();
    job->lend_until = t1 + (t1 - t0);
    std::lock_guard<std::mutex> lk(job->mu);
    job->lent_jobs += ran;
    job->lent_ms += t1 - t0;
}

// ---- the fit launches of an ARIMA pass ----------------------------------------------------------------------------------
// A pass's fit (fit_solo, or fit_beside for a job run in another fit's yield) is enqueued on ctx->stream behind the reset
// of its words and fit_ev[0], and waited for without blocking behind it (wait_fit): the worker polls, every millisecond,
// an event recorded after the kernel, and watches each part of the launch in flight -- one for a job's own fit or resume,
// two for a joint launch: b, the job fitting beside a yielded fit, and a, that fit.  Its copies and word writes run on the
// copy stream, beside the kernel:
//   cancel: a cancel of a part's job writes 1 into the part's cancel word (one GPU only: on several GPUs the fit reads the
//     stop board, which tad_cancel writes itself, post_stop).  A cancel of b makes a leave too (2), so b fails at once; a
//     cancelled a fails once b has ended, like any parked job;
//   end: once every fit of b is counted done and a is clear, 2 goes into a's word: its part leaves within one evaluation
//     round, its resume points written.  A part is clear when it is cancelled or has finished again every fit its last
//     leave dropped (so none is dropped twice);
//   yield (fit sharing, tad_set_fit_sharing): once the job whose wait this is (the solo job, or b) can yield (share), is
//     neither cancelled nor yielded in this launch, a has not been told to leave, every part is clear, the job's quiet
//     time has passed and a job is waiting that interleave() would run, 2 goes into every part's word that holds neither
//     1 nor 2.  Once the kernel has left, the pass is parked, the waiting jobs run (park_pass), and the rest of the fit is
//     launched: the solo fit's resume (launch_arima_resume) or the next joint launch.  Fairness: after a resume the fit
//     does not yield again until every fit the last yield dropped has finished again and it has run at least as long as
//     that interleave took (job->quiet_until).  So the work yields throw away is at most one fitting of each prefix, and
//     under a steady stream of short jobs the fit phase (parked time left out) takes at most about twice as long;
//   counts: the parts' counters come back every 50 ms for a solo fit, every poll during a joint launch or while a part
//     has a redo pending, and are published added to each job's counts before the pass (tad_job_progress).
// Once the kernel has ended the final counts are published and each part's fits dropped read; a's part in joint launches
// is fit time for a, not parked time.  Returns whether the launch yielded: the fit has fits left, and the pass is parked
// before its next launch.
bool wait_fit(tad_ctx *ctx, YieldedFit &own, YieldedFit *a)
{
    struct Watch {
        YieldedFit *f;
        tad_ctx::FitWords *h;
        uint32_t redone = 0;             // of the fits f's last leave dropped, those finished again (as last copied back)
        bool cancelled = false, left = false;   // 1 / 2 written into its cancel word in this launch
        bool redoing() const { return redone < f->dropped; }
        bool clear() const { return cancelled || !redoing(); }
        uint32_t *redo() const { return f->part.resume + 2 * (size_t)f->part.S; }
    };
    tad_ctx::FitPinned *H = ctx->h_fit;
    const int n = a ? 2 : 1;
    Watch w[2] = {{&own, &H->part[0]}, {a, &H->part[1]}};
    auto word = [&](Watch &p, const uint32_t *value) {
        CU(cudaMemcpyAsync(p.f->part.cancel, value, 4, cudaMemcpyHostToDevice, ctx->copy_stream));
    };
    auto leave = [&](Watch &p) {
        if (!p.cancelled && !p.left) word(p, &H->leave);
        p.left = true;
    };
    auto publish = [](const YieldedFit *f, const tad_ctx::FitCounts &c) {
        std::lock_guard<std::mutex> lk(f->job->mu);
        f->job->prog.fits_total = f->total0 + c.total;
        f->job->prog.fits_done = f->done0 + c.done;
    };
    const bool cancellable = ctx->cfg.world_size == 1;
    const double t_launch = now_ms();
    double next_copy = t_launch, t_word = 0;
    bool copying = false, counted = false;
    CU(cudaEventRecord(ctx->fit_ev[1], ctx->stream));
    for (;;) {
        for (int i = n - 1; i >= 0; i--)
            if (cancellable && !w[i].cancelled && w[i].f->job->cancel.load()) {
                word(w[i], &H->cancel);
                w[i].cancelled = true;
                if (i == 0 && a) leave(w[1]);
            }
        if (a && counted && !w[1].left && !w[1].cancelled && w[1].clear() && w[0].h->run.done == w[0].h->run.total)
            leave(w[1]);
        if (own.job->share && !w[0].cancelled && !w[0].left && !w[1].left && w[0].clear() && (!a || w[1].clear()) &&
            now_ms() >= own.job->quiet_until && interleave_waiting(ctx, own.job)) {
            for (int i = 0; i < n; i++) leave(w[i]);
            t_word = now_ms();
        }
        const cudaError_t e = cudaEventQuery(ctx->fit_ev[1]);
        if (e != cudaErrorNotReady) {
            CU(e);
            break;
        }
        if (copying) {
            const cudaError_t c = cudaEventQuery(ctx->fits_ev);
            if (c != cudaErrorNotReady) {
                CU(c);
                for (int i = 0; i < n; i++) {
                    publish(w[i].f, w[i].h->run);
                    if (w[i].redoing()) w[i].redone = w[i].h->redone;
                }
                counted = true;
                copying = false;
            }
        }
        if (!copying && (a || w[0].redoing() || now_ms() >= next_copy)) {
            for (int i = 0; i < n; i++) {
                CU(cudaMemcpyAsync(&w[i].h->run, w[i].f->part.fits_total, 8, cudaMemcpyDeviceToHost, ctx->copy_stream));
                if (w[i].redoing())
                    CU(cudaMemcpyAsync(&w[i].h->redone, w[i].redo() + 1, 4, cudaMemcpyDeviceToHost, ctx->copy_stream));
            }
            CU(cudaEventRecord(ctx->fits_ev, ctx->copy_stream));
            copying = true;
            next_copy = now_ms() + 50.0;
        }
        std::this_thread::sleep_for(std::chrono::milliseconds(1));
    }
    CU(cudaStreamSynchronize(ctx->copy_stream));            // no copy or word write is left behind the kernel
    for (int i = 0; i < n; i++) {
        CU(cudaMemcpyAsync(&w[i].h->end, w[i].f->part.fits_total, 8, cudaMemcpyDeviceToHost, ctx->stream));
        if (w[i].f->part.resume) CU(cudaMemcpyAsync(&w[i].h->dropped, w[i].redo(), 4, cudaMemcpyDeviceToHost, ctx->stream));
    }
    CU(cudaStreamSynchronize(ctx->stream));
    const double t_end = now_ms();
    for (int i = 0; i < n; i++) {
        publish(w[i].f, w[i].h->end);
        if (w[i].f->part.resume) w[i].f->dropped = w[i].h->dropped;
    }
    if (a) a->fit_ms += t_end - t_launch;
    // not yielded, cancelled (the caller fails the job), or every fit finished before the kernel saw the word
    const bool yielded = w[0].left && !w[0].cancelled && w[0].h->end.done != w[0].h->end.total;
    if (yielded && getenv("TAD_DEBUG_YIELD"))
        fprintf(stderr, "yield: kernel left %.2f ms after the word, %u + %u fits dropped\n", t_end - t_word, own.dropped,
                a ? a->dropped : 0u);
    return yielded;
}

// Before a fit launch: the cancel and redo words the last launch of p and q left are zeroed (null: none to zero), and the
// copy stream's reads and writes of the fit's words wait for that (fit_ev[0]).
void arm_fit(tad_ctx *ctx, const FitPart *p, const FitPart *q = nullptr)
{
    for (const FitPart *r : {p, q})
        if (r) {
            CU(cudaMemsetAsync(r->cancel, 0, 4, ctx->stream));
            CU(cudaMemsetAsync(r->resume + 2 * (size_t)r->S, 0, 8, ctx->stream));
        }
    CU(cudaEventRecord(ctx->fit_ev[0], ctx->stream));
    CU(cudaStreamWaitEvent(ctx->copy_stream, ctx->fit_ev[0], 0));
}

// After a launch has yielded: the pass of `job` is parked while the waiting jobs run (interleave); yf: its fit, which an
// ARIMA job run there may fit beside.  Returns the time parked, yf's part of joint launches left out; the fit does not
// yield again before it has run as long.
double park_pass(tad_ctx *ctx, tad_job *job, YieldedFit *yf)
{
    if (yf) yf->fit_ms = 0;
    const double t0 = now_ms();
    interleave(ctx, job, yf);
    const double t1 = now_ms();
    const double away = std::max(0.0, t1 - t0 - (yf ? yf->fit_ms : 0.0));
    job->quiet_until = t1 + away;
    std::lock_guard<std::mutex> lk(job->mu);
    job->yields++;
    job->parked_ms += away;
    return away;
}

// A pass's own fit: launch_arima_fit, then after each yield the resume of what is left.  Returns the time parked (ms).
double fit_solo(tad_ctx *ctx, YieldedFit &fit, const uint64_t *csr_v, uint64_t &launches)
{
    arm_fit(ctx, nullptr);
    CU(launch_arima_fit(ctx->stream, fit.part, csr_v, ctx->cfg.world_size > 1 ? ctx->board : nullptr, fit.job->ordinal));
    launches += 2;
    double parked = 0;
    while (wait_fit(ctx, fit, nullptr)) {
        parked += park_pass(ctx, fit.job, &fit);
        arm_fit(ctx, &fit.part);
        CU(launch_arima_resume(ctx->stream, fit.part));
        launches++;
    }
    return parked;
}

// The fit of b, an ARIMA job run in the yield of the fit a (TAD_FLAG_FIT_BESIDE): Box-Cox, then joint launches of b's
// series beside those a has left, from a's lowest unfinished series, until b's fit has ended.  After a yield of b only
// b's pass is parked (one level deeper, EWMA and DBSCAN jobs only).  d_from: a device word of scratch.  Returns the time
// b's pass was parked (ms).
double fit_beside(tad_ctx *ctx, YieldedFit &b, YieldedFit &a, const uint64_t *csr_v, uint32_t *d_from, uint64_t &launches)
{
    cudaStream_t st = ctx->stream;
    CU(launch_arima_boxcox(st, b.part, csr_v));             // b's fit count is final before the joint launch
    launches++;
    double parked = 0;
    for (bool first = true;; first = false) {
        CU(launch_arima_unfinished(st, a.part, d_from));
        launches++;
        CU(cudaMemcpyAsync(&ctx->h_fit->from, d_from, 4, cudaMemcpyDeviceToHost, st));
        CU(cudaStreamSynchronize(st));
        const uint32_t lo = ctx->h_fit->from;               // ~0u: a has no fits left
        arm_fit(ctx, &a.part, first ? nullptr : &b.part);
        CU(launch_arima_pair(st, a.part, lo == ~0u ? 0 : lo, lo == ~0u ? 0 : a.part.S - lo, b.part, first));
        launches++;
        if (!wait_fit(ctx, b, &a)) return parked;
        parked += park_pass(ctx, b.job, nullptr);
    }
}

int pick_logb(const tad_ctx *ctx, uint64_t rows)
{
    if (ctx->debug_logb >= 0) return ctx->debug_logb;
    // mean bucket ~ 0.375 * capacity: connection sizes are lumpy, so leave head-room
    // 4 ranks and more: twice the rows per bucket -- half as many, twice as large pieces for the peer pull (small scattered
    // remote reads are what limits the pulled group phase); every rank derives the same value from the same world size
    uint64_t target = (uint64_t)kGroupTarget * (ctx->cfg.world_size >= 4 ? 2 : 1);
    if (ctx->debug_target > 0) target = (uint64_t)ctx->debug_target;
    int logb = 0;
    while (logb < 22 && (rows >> logb) > target) logb++;
    return logb;
}

size_t col_bytes(int idx, uint64_t rows)
{
    static const size_t w[10] = {4, 4, 2, 2, 1, 4, 4, 8, 4, 4};
    return w[idx] * rows;
}

void *col_ptr(const tad_columns &c, int idx)
{
    switch (idx) {
    case 0: return c.src_ip;
    case 1: return c.dst_ip;
    case 2: return c.src_port;
    case 3: return c.dst_port;
    case 4: return c.proto;
    case 5: return c.flow_start;
    case 6: return c.flow_end;
    case 7: return c.value;
    case 8: return c.src_ns;
    default: return c.dst_ns;
    }
}

void set_col(ColPtrs &c, int i, const void *p)
{
    switch (i) {
    case 0: c.src_ip = (const uint32_t *)p; break;
    case 1: c.dst_ip = (const uint32_t *)p; break;
    case 2: c.src_port = (const uint16_t *)p; break;
    case 3: c.dst_port = (const uint16_t *)p; break;
    case 4: c.proto = (const uint8_t *)p; break;
    case 5: c.flow_start = (const uint32_t *)p; break;
    case 6: c.flow_end = (const uint32_t *)p; break;
    case 7: c.value = (const uint64_t *)p; break;
    case 8: c.src_ns = (const uint32_t *)p; break;
    default: c.dst_ns = (const uint32_t *)p; break;
    }
}

// A rank stream job whose first round was empty takes its peers' column set `mask` (run_passes_multi), so that it holds
// the pass columns they hold; the pointers stand for columns of no rows and are never read.
void adopt_columns(tad_job *job, uint64_t mask)
{
    static uint64_t none = 0;
    std::lock_guard<std::mutex> lk(job->mu);
    if (job->in.pushed) return;
    tad_columns &c = job->cols;
    void **slot[10] = {(void **)&c.src_ip, (void **)&c.dst_ip, (void **)&c.src_port, (void **)&c.dst_port, (void **)&c.proto,
                       (void **)&c.flow_start, (void **)&c.flow_end, (void **)&c.value, (void **)&c.src_ns, (void **)&c.dst_ns};
    for (int i = 0; i < 10; i++)
        if (mask >> i & 1) *slot[i] = &none;
}

// Whether column i of a job's blocks arrives as text: a key slot (src_ip, dst_ip) or a namespace slot (src_ns, dst_ns).
bool is_text(const tad_job *job, int i) { return i < 2 ? job->text[i] : i >= 8 && job->text[i - 6]; }

// Whether a job's rows carry column i: its first block's column, or a text slot encoded (or tested) into it on the device.
bool has_col(const tad_job *job, int i) { return col_ptr(job->cols, i) || is_text(job, i); }

// A block's columns as kernel input.
ColPtrs col_ptrs(const tad_columns &b)
{
    ColPtrs c{};
    for (int i = 0; i < 10; i++) set_col(c, i, col_ptr(b, i));
    return c;
}

// The columns from row `lo` on.
ColPtrs offset_cols(ColPtrs c, uint64_t lo)
{
    auto at = [lo](auto *&p) { if (p) p += lo; };
    at(c.src_ip); at(c.dst_ip); at(c.src_port); at(c.dst_port); at(c.proto);
    at(c.flow_start); at(c.flow_end); at(c.value); at(c.src_ns); at(c.dst_ns);
    return c;
}

// The job's time window and ns_ignore list as the kernels' row filter.  `ns`: the rows carry a namespace column, so a
// non-empty list is uploaded.
RowFilter row_filter(tad_ctx *ctx, const tad_job *job, bool ns)
{
    RowFilter f{};
    f.start_time = job->spec.start_time;
    f.end_time = job->spec.end_time;
    if (ns && !job->ns_ignore.empty()) {
        ensure(ctx, ctx->ns_ignore, job->ns_ignore.size() * 4);
        CU(cudaMemcpyAsync(ctx->ns_ignore.p, job->ns_ignore.data(), job->ns_ignore.size() * 4, cudaMemcpyHostToDevice,
                           ctx->stream));
        f.n_ns_ignore = (uint32_t)job->ns_ignore.size();
        f.ns_ignore = static_cast<const uint32_t *>(ctx->ns_ignore.p);
    }
    return f;
}

struct OutLayout {
    size_t off[11];
    size_t total;
};
// src_ip dst_ip flow_start flow_end (u32) | stddev algo_calc throughput (f64) | ports (u16) | proto anomaly (u8)
OutLayout out_layout(uint64_t cap)
{
    OutLayout L;
    size_t o = 0;
    auto add = [&](int i, size_t w) {
        L.off[i] = o;
        o += (w * cap + 255) & ~size_t(255);
    };
    add(0, 8); add(1, 8); add(2, 8);          // stddev, algo_calc, throughput
    add(3, 4); add(4, 4); add(5, 4); add(6, 4);  // src_ip, dst_ip, flow_start, flow_end
    add(7, 2); add(8, 2);                      // src_port, dst_port
    add(9, 1); add(10, 1);                     // proto, anomaly
    L.total = o;
    return L;
}

OutCols out_cols(void *base, const OutLayout &L)
{
    char *b = static_cast<char *>(base);
    OutCols o;
    o.stddev = reinterpret_cast<double *>(b + L.off[0]);
    o.algo_calc = reinterpret_cast<double *>(b + L.off[1]);
    o.throughput = reinterpret_cast<double *>(b + L.off[2]);
    o.src_ip = reinterpret_cast<uint32_t *>(b + L.off[3]);
    o.dst_ip = reinterpret_cast<uint32_t *>(b + L.off[4]);
    o.flow_start = reinterpret_cast<uint32_t *>(b + L.off[5]);
    o.flow_end = reinterpret_cast<uint32_t *>(b + L.off[6]);
    o.src_port = reinterpret_cast<uint16_t *>(b + L.off[7]);
    o.dst_port = reinterpret_cast<uint16_t *>(b + L.off[8]);
    o.proto = reinterpret_cast<uint8_t *>(b + L.off[9]);
    o.anomaly = reinterpret_cast<uint8_t *>(b + L.off[10]);
    return o;
}

// first guess of the result capacity; detect reruns with the exact count when more rows are flagged
uint64_t out_cap_guess(uint64_t points, bool emit_all)
{
    uint64_t out_cap = emit_all ? points : (points / 8 + (1u << 16));
    if (out_cap > points) out_cap = points;
    return out_cap ? out_cap : 1;
}

// Device bytes of every workspace buffer one single-GPU pipeline run sizes from its shape: the one description of the
// layout.  run_pipeline() sizes its buffers from it (with the counts it knows at each stage) and the planner sums it with
// upper bounds (rows for owned rows, series and points).  Not in it: the spill scratch (known after grouping), a detect
// rerun's larger result buffer, and buffers of a few KB (kFixedBytes).
struct PipeShape {
    uint64_t rows = 0;               // input rows
    const tad_columns *host = nullptr;   // host input: the columns copied to d_col[]
    int algo = TAD_ALGO_EWMA;
    uint32_t B = 1, Bl = 1;          // buckets; buckets this GPU owns
    bool optimistic = false;         // fixed-capacity bucket slots instead of the exact partition
    bool resume = false;             // an ARIMA fit that can yield: its resume points (tad_set_fit_sharing)
    uint64_t owned = 0, series = 0, out_cap = 1;
};
struct PipeSizes {
    size_t col[10], part, slots, ovf, entries, hist, offsets, cursor, big_list, big_base, cls_list, nsb, npb, csr_v, csr_t,
        csr_p, sbase, outb, dbx, dbi, ar_y, ar_pred, ar_lam, ar_res;
};
constexpr size_t kOutWidth[11] = {8, 8, 8, 4, 4, 4, 4, 2, 2, 1, 1};   // bytes per result row of each out_layout column
constexpr uint64_t kBudgetHeadroom = 512ull << 20; // default budget: device memory left free for the CUDA context and others
constexpr size_t kFixedBytes = 1u << 20;        // stats, scan flags, ns_ignore list, small staging
constexpr uint64_t kSlotBudget = 40ull << 30;   // optimistic slot buffer at most half of an 80 GB H100

PipeSizes pipe_sizes(const PipeShape &s)
{
    PipeSizes z{};
    for (int i = 0; i < 10; i++) z.col[i] = s.host && col_ptr(*s.host, i) ? col_bytes(i, s.rows) : 0;
    const size_t B = s.B, cap_rows = s.owned ? s.owned : 1;
    z.part = (s.rows ? s.rows : 1) * sizeof(Row32);
    z.slots = s.optimistic ? B * kGroupCap * sizeof(Row32) : 0;
    z.ovf = s.optimistic ? std::max<uint64_t>(1u << 20, s.rows / 32) * sizeof(Row32) : 0;
    z.entries = s.optimistic ? cap_rows * sizeof(SeriesEntry) : 0;
    z.hist = z.cursor = z.big_list = B * 4;
    z.nsb = z.npb = (size_t)s.Bl * 4;
    z.offsets = z.big_base = (B + 1) * 4;
    z.cls_list = B * 4 * kGroupClasses;
    z.csr_v = cap_rows * 8 + 64;       // + one sector: the direct detector reads whole 32-byte sectors
    z.csr_t = cap_rows * 4;
    z.csr_p = z.dbx = s.algo == TAD_ALGO_DBSCAN ? cap_rows * 4 : 0;
    z.dbi = s.algo == TAD_ALGO_DBSCAN ? cap_rows : 0;
    z.sbase = sbase_words(s.B, cap_rows) * 4;
    z.outb = out_layout(s.out_cap).total;
    z.ar_y = z.ar_pred = s.algo == TAD_ALGO_ARIMA ? cap_rows * 8 : 0;
    z.ar_lam = s.algo == TAD_ALGO_ARIMA ? ((size_t)s.series + 1) * 8 : 0;
    z.ar_res = s.algo == TAD_ALGO_ARIMA && s.resume ? ((size_t)s.series + 1) * 8 : 0;
    return z;
}

// (buffer, bytes) of every buffer in PipeSizes
std::vector<std::pair<DevBuf *, size_t>> pipe_bufs(tad_ctx *ctx, const PipeSizes &z)
{
    std::vector<std::pair<DevBuf *, size_t>> v = {
        {&ctx->part, std::max(z.part, z.slots)}, {&ctx->ovf, z.ovf}, {&ctx->entries, z.entries}, {&ctx->hist, z.hist},
        {&ctx->offsets, z.offsets}, {&ctx->cursor, z.cursor}, {&ctx->big_list, z.big_list}, {&ctx->big_base, z.big_base},
        {&ctx->cls_list, z.cls_list}, {&ctx->nsb, z.nsb}, {&ctx->npb, z.npb}, {&ctx->csr_v, z.csr_v}, {&ctx->csr_t, z.csr_t},
        {&ctx->csr_p, z.csr_p}, {&ctx->sbase, z.sbase}, {&ctx->outb, z.outb}, {&ctx->dbx, z.dbx}, {&ctx->dbi, z.dbi},
        {&ctx->ar_y, z.ar_y}, {&ctx->ar_pred, z.ar_pred}, {&ctx->ar_lam, z.ar_lam}, {&ctx->ar_res, z.ar_res}};
    for (int i = 0; i < 10; i++) v.push_back({&ctx->d_col[i], z.col[i]});
    return v;
}

// Workspace the context holds once every listed buffer has grown to its size: `held` plus the growth, each buffer sized
// as ensure() sizes it.  With `held` = 0 and empty buffers (fresh = true): the need of a job on an empty workspace.
size_t workspace_after(tad_ctx *ctx, const std::vector<std::pair<DevBuf *, size_t>> &bufs, bool fresh)
{
    size_t total = (fresh ? 0 : ctx->held) + kFixedBytes;
    for (const auto &b : bufs) {
        const size_t cap = fresh ? 0 : b.first->cap;
        if (b.second > cap) total += alloc_bytes(b.second) - cap;
    }
    return total;
}

// ---- partition decisions of run_pipeline, which the planners share ----------------------------------------------------
// On several GPUs they depend only on values every rank shares (the global rows, the job, the world size and the run-time
// switches every rank must see alike), so every rank computes them for every other rank.
int log_world(const tad_ctx *ctx)
{
    int l = 0;
    while ((1 << l) < ctx->cfg.world_size) l++;
    return l;
}

uint32_t buckets(const tad_ctx *ctx, uint64_t global)      // global buckets; a rank owns B >> log_world of them
{
    return 1u << std::max(pick_logb(ctx, global), log_world(ctx));
}

// Whether one GPU takes the optimistic partition: its slot buffer at most half of an 80 GB H100 (kSlotBudget).
bool one_gpu_optimistic(const tad_ctx *ctx, uint64_t rows, uint64_t B)
{
    return ctx->optimistic && rows > 0 && B * kGroupCap * sizeof(Row32) <= kSlotBudget;
}

// Multi-GPU slot rows of a bucket: a source holds 1/world of a bucket on average.
uint32_t slot(const tad_ctx *ctx) { return std::max<uint32_t>(256u, (uint32_t)kGroupCap / (uint32_t)ctx->cfg.world_size); }
// The exported buffer's arrival counters of B buckets, padded; the rows follow them.
size_t xbuf_cnt_bytes(uint64_t B) { return (B * 4 + 65535) & ~size_t(65535); }
size_t slot_xbuf_bytes(const tad_ctx *ctx, uint64_t B) { return xbuf_cnt_bytes(B) + B * slot(ctx) * sizeof(Row32); }

// Whether several GPUs may take the optimistic slot path for `global` rows.
bool slots_allowed(const tad_ctx *ctx, uint64_t global)
{
    const uint64_t B = buckets(ctx, global);
    return ctx->peer_pull && ctx->optimistic && global > 0 && B * slot(ctx) <= (1ull << 31) &&
           slot_xbuf_bytes(ctx, B) <= ctx->x_budget;
}

// Exported-buffer bytes for `global` rows: the exact partition pulled by the peers (every rank's buffer holds the largest
// shard, `max_rows`) and, with `slots`, the optimistic slots of all B buckets.
size_t xbuf_bytes(const tad_ctx *ctx, uint64_t global, uint64_t max_rows, bool slots)
{
    const uint64_t B = buckets(ctx, global);
    size_t x = ctx->peer_pull && ctx->exact_pull ? xbuf_cnt_bytes(B) + std::max<uint64_t>(max_rows, 1) * sizeof(Row32) : 0;
    if (slots && slots_allowed(ctx, global)) x = std::max(x, slot_xbuf_bytes(ctx, B));
    return x;
}

// The multi-GPU exact partition's buffers for K row chunks per rank, in the order run_pipeline grows them.
std::vector<std::pair<DevBuf *, size_t>> exact_bufs(tad_ctx *ctx, size_t B, size_t Bl, size_t K)
{
    const size_t NS = (size_t)ctx->cfg.world_size * K;      // segments: (source rank, chunk)
    return {{&ctx->hist, B * 4 * K}, {&ctx->offsets, (B + 1) * 4 * K}, {&ctx->cursor, B * 4 * K},
            {&ctx->hist_all, B * 4 * NS}, {&ctx->seg_off, (Bl + 1) * 4 * NS}, {&ctx->seg_total, Bl * 4}};
}

// ---- collectives through the small scratch (tad_ctx::kSmallWords) ----------------------------------------------------
// Blocking all-gather of h_small[0, n) of every rank into h_small[n, n + n * world) on ctx->stream.  `timed`: returns the
// collective's time in ms (the ranks' arrival skew), measured with ctx->ev[0..1]; else 0.
float gather_small(tad_ctx *ctx, int n, bool timed)
{
    cudaStream_t st = ctx->stream;
    unsigned long long *d_small = static_cast<unsigned long long *>(ctx->small.p);
    CU(cudaMemcpyAsync(d_small, ctx->h_small, n * 8, cudaMemcpyHostToDevice, st));
    if (timed) CU(cudaEventRecord(ctx->ev[0], st));
    if (nccl_allgather(&ctx->nccl, d_small, d_small + n, n * 8, st)) fail(TAD_ERR_NCCL, "%s", nccl_last_error());
    if (timed) CU(cudaEventRecord(ctx->ev[1], st));
    CU(cudaMemcpyAsync(ctx->h_small + n, d_small + n, (size_t)n * 8 * ctx->cfg.world_size, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    float ms = 0;
    if (timed) CU(cudaEventElapsedTime(&ms, ctx->ev[0], ctx->ev[1]));
    return ms;
}

// Barrier of the ranks on ctx->stream (an 8-byte all-gather); nccl_allgather's return code.
int peer_barrier(tad_ctx *ctx)
{
    unsigned long long *d_small = static_cast<unsigned long long *>(ctx->small.p);
    return nccl_allgather(&ctx->nccl, d_small + tad_ctx::kWBarrier, d_small + tad_ctx::kWBarrierIn, 8, ctx->stream);
}

// Unmaps every peer's exported buffer; the first error.
cudaError_t unmap_peers(tad_ctx *ctx)
{
    cudaError_t err = cudaSuccess;
    for (void *&p : ctx->peer_x) {
        const cudaError_t e = p ? nccl_ipc_unmap(&ctx->nccl, p) : cudaSuccess;
        if (err == cudaSuccess) err = e;
        p = nullptr;
    }
    ctx->peers_mapped = false;
    return err;
}

// ---- cancel on several GPUs (DESIGN.md section 6) ------------------------------------------------------------------------
// Maps every peer's stop board (the first job of a multi-GPU context: every rank runs it, so every rank meets here).
// Without peer pull (TAD_PEER_PULL=0) a rank exports nothing, and a board that fails to map is left out: a cancel then
// reaches only the boards that are mapped, and the ranks whose fits it does not stop fail at the verdict.
void share_boards(tad_ctx *ctx)
{
    constexpr int G = tad_ctx::kGatherMax;
    const int me = ctx->cfg.rank;
    ensure(ctx, ctx->small, tad_ctx::kSmallDevWords * 8);
    memset(ctx->h_small, 0, G * 8);
    ctx->h_small[0] = ctx->peer_pull ? 1 : 0;
    if (ctx->peer_pull) CU(nccl_ipc_export(&ctx->nccl, ctx->board, ctx->h_small + 2));      // a 64-byte handle in words 2..9
    gather_small(ctx, G, false);
    uint32_t *mapped[kMaxRanks] = {};
    for (int r = 0; r < ctx->cfg.world_size; r++) {
        if (r == me || !ctx->peer_pull || !ctx->h_small[G * (1 + r)]) continue;
        void *p = nullptr;
        if (nccl_ipc_map(&ctx->nccl, ctx->h_small + G * (1 + r) + 2, &p) == cudaSuccess) mapped[r] = static_cast<uint32_t *>(p);
        else cudaGetLastError();
    }
    std::lock_guard<std::mutex> lk(ctx->board_mu);
    for (int r = 0; r < ctx->cfg.world_size; r++)
        if (r != me) ctx->peer_board[r] = mapped[r];
    ctx->boards_shared = true;
}

// Writes `ordinal` into this rank's word of every board it has mapped, its own included, so that the fit of that job
// stops on every rank within one evaluation round.  Called under the cancelled job's `mu`, from tad_cancel or tad_release
// while the job runs, or by the worker as it takes a job cancelled in the queue.  The copies run on board_stream, so the
// write waits for no job's work (the worker may be blocked in a collective or waiting for the loopback device turn), and
// the calling thread's current device is left as it was.  A word only grows: the write of a job that precedes the last
// one written is dropped, so a stop for job k never stops another job.
void post_stop(tad_ctx *ctx, uint32_t ordinal)
{
    std::lock_guard<std::mutex> lk(ctx->board_mu);
    if (!ctx->board || ordinal <= ctx->h_board[0]) return;
    int dev = -1;
    if (cudaGetDevice(&dev) != cudaSuccess) dev = -1;
    if (cudaSetDevice(ctx->cfg.device) != cudaSuccess) return;
    ctx->h_board[0] = ordinal;
    cudaError_t e = cudaSuccess;
    for (int r = 0; r < ctx->cfg.world_size; r++)
        if (ctx->peer_board[r] && e == cudaSuccess)
            e = cudaMemcpyAsync(ctx->peer_board[r] + ctx->cfg.rank, ctx->h_board, 4, cudaMemcpyDefault, ctx->board_stream);
    if (cudaStreamSynchronize(ctx->board_stream) != cudaSuccess || e != cudaSuccess)
        cudaGetLastError();      // a write that did not land: the verdict still fails the job on every rank
    if (dev >= 0) cudaSetDevice(dev);
}

// A multi-GPU cancel of `job` by tad_cancel or tad_release (under job->mu): the stop board is written while the worker
// runs the job; a queued job's is written as the worker takes it (run_job).
void stop_running(tad_job *job)
{
    const int s = job->st.state;
    if (job->ctx && job->ctx->cfg.world_size > 1 && job->started && s != TAD_STATE_COMPLETED && s != TAD_STATE_FAILED)
        post_stop(job->ctx, job->ordinal);
}

// After a multi-GPU fit that left with fits undone: the rank whose board word holds this job's ordinal (kMaxRanks: none).
int board_stopper(tad_ctx *ctx, const tad_job *job)
{
    CU(cudaMemcpyAsync(ctx->h_board + 8, ctx->board, 4 * kMaxRanks, cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
    for (int r = 0; r < ctx->cfg.world_size; r++)
        if (ctx->h_board[8 + r] == job->ordinal) return r;
    return kMaxRanks;
}

// The agreed points of a multi-GPU job -- the verdict all-gather that ends it and, in hash-range passes, the end of every
// pass -- carry one 8-byte word per rank: 2 its job was cancelled there (its own flag, read once); 4 its fit stopped on
// the board, with bits 8.. the rank whose word stopped it (kMaxRanks: none); bit 0 is the pass driver's split.  A rank
// that cancelled after its flag was read can still stop a peer's fit that is running, so a stopped fit fails the job
// even where no rank flags the cancel; and every rank decides on the same gathered words.
uint64_t stop_word(const tad_job *job, int fit_stop)
{
    return (job->cancel.load() ? 2u : 0u) | (fit_stop >= 0 ? 4u | ((uint64_t)fit_stop << 8) : 0u);
}

// A rank stream job between two blocks: the rank whose stop for `job` is on this rank's board (-1: none).  Read on
// board_stream, so the job's work in flight is not waited for.
int board_stop(tad_ctx *ctx, const tad_job *job)
{
    std::lock_guard<std::mutex> lk(ctx->board_mu);
    CU(cudaMemcpyAsync(ctx->h_board + 8, ctx->board, 4 * kMaxRanks, cudaMemcpyDeviceToHost, ctx->board_stream));
    CU(cudaStreamSynchronize(ctx->board_stream));
    for (int r = 0; r < ctx->cfg.world_size; r++)
        if (ctx->h_board[8 + r] == job->ordinal) return r;
    return -1;
}

bool any_stop(const unsigned long long *w, int world)
{
    for (int r = 0; r < world; r++)
        if (w[r] & 6) return true;
    return false;
}

// Fails the job alike on every rank when a word of `w` (one per rank) carries a cancel or a stopped fit: TAD_ERR_CANCELLED
// naming the first rank that cancelled, TAD_ERR_INTERNAL for a fit stopped with no board word holding the job's ordinal.
void agree_stop(const unsigned long long *w, int world)
{
    for (int r = 0; r < world; r++)
        if (w[r] & 2) fail(TAD_ERR_CANCELLED, "job cancelled (rank %d)", r);
    for (int r = 0; r < world; r++) {
        if (!(w[r] & 4)) continue;
        const int by = (int)((w[r] >> 8) & 0xff);
        if (by >= world) fail(TAD_ERR_INTERNAL, "rank %d: the ARIMA fit stopped with no cancel on any rank", r);
        fail(TAD_ERR_CANCELLED, "job cancelled (rank %d)", by);
    }
}

// Fails a rank stream job alike on every rank when a word of `w` (one per rank) carries an input verdict (run_passes_multi):
// bits 40.., a block that rank refused (its error code, negated); bit 32, a later round whose per-residue counts differ
// from that rank's first round's.
void agree_input(const tad_job *job, const unsigned long long *w, int world, int me)
{
    for (int r = 0; r < world; r++) {
        const int code = -(int)((w[r] >> 40) & 0xff);
        if (code == TAD_ERR_UNSUPPORTED)
            fail(code, "rank %d: text key columns are not supported on a job streamed to several GPUs", r);
        if (code) fail(code, "rank %d: %s", r, r == me ? job->in.msg : "a block of its stream was refused");
    }
    for (int r = 0; r < world; r++)
        if (w[r] >> 32 & 1)
            fail(TAD_ERR_INVALID_ARG, "rank %d: a round delivered other per-residue row counts than its first round: the "
                 "source changed between reads", r);
}

// Result of one pipeline run: a one-pass job or one hash-range pass.
struct PassOut {
    uint64_t kept = 0, owned = 0, points = 0, series = 0, out_rows = 0, spill_rows = 0, launches = 0;
    double phase_ms[TAD_NPHASES] = {0};
    double device_ms = 0;
    PinnedBlock block;               // result rows, out_layout(out_rows) in pinned host memory
    int fit_stop = -1;               // multi-GPU ARIMA: the fit stopped on the board, by this rank's word (board_stopper)
};

// The pipeline (ingest, partition, exchange, group, detect, egress) over `hc`.  `filters`: apply the job's time window
// and ns_ignore list (passes were filtered by the split kernel already).  `force_exact`: the exact partition even where
// the optimistic slot buffer would be used (the planner found it does not fit the budget).
// `pass`: one pass of a multi-GPU job in passes (run_passes_multi), null otherwise.  Its sizes come from the all-gathered
// counts, so they are the same on every rank: the bucket count follows its global rows and the NCCL exchange's chunk count
// its largest shard.  The pipeline then leaves every decision that changes which collectives a rank issues to the
// driver's end-of-pass all-gather: a cancel or a stopped fit does not throw here, and the peer-pull end barrier is that
// all-gather, so a rank that throws PassSplit has issued every collective its peers have.  Outside passes a multi-GPU job
// ends with the verdict all-gather, which takes those decisions the same way.
struct AgreedPass {
    uint64_t global_rows;            // the pass's rows over all ranks
    uint64_t max_rows;               // the most rows one rank holds in the pass
};
void run_pipeline(tad_ctx *ctx, tad_job *job, const tad_columns &hc, bool filters, bool force_exact, PassOut &out,
                  const AgreedPass *pass = nullptr)
{
    const tad_job_spec &sp = job->spec;
    const uint64_t R = hc.rows;
    cudaStream_t st = ctx->stream;
    uint64_t launches = 0;
    int nev = 0;
    int ev_phase[kMaxEvents];
    auto mark = [&](int phase) {          // event closing `phase`
        if (nev < kMaxEvents) {
            CU(cudaEventRecord(ctx->ev[nev], st));
            ev_phase[nev++] = phase;
        }
    };
    auto check_cancel = [&]() {          // several GPUs: a cancel acts at the verdict, where every rank decides alike
        if (ctx->cfg.world_size == 1 && job->cancel.load()) fail(TAD_ERR_CANCELLED, "job cancelled");
    };

    CU(cudaSetDevice(ctx->cfg.device));
    set_progress(job, TAD_STATE_RUNNING, 0);
    ensure(ctx, ctx->stats, 64 * sizeof(uint32_t));
    uint32_t *d_stats = static_cast<uint32_t *>(ctx->stats.p);
    CU(cudaMemsetAsync(d_stats, 0, 64 * sizeof(uint32_t), st));
    auto read_stats = [&]() {             // the device scalars -> h_stats, with everything enqueued before
        CU(cudaMemcpyAsync(ctx->h_stats, d_stats, ST_COUNT * 4, cudaMemcpyDeviceToHost, st));
        CU(cudaStreamSynchronize(st));
    };
    if (!ctx->scan_sync.p) {
        ensure(ctx, ctx->scan_sync, scan_sync_bytes());
        CU(cudaMemsetAsync(ctx->scan_sync.p, 0, scan_sync_bytes(), st));
    }

    // ---- ingest: host columns -> device (device-resident columns are used in place) -------
    // Host input is copied in chunks on a second stream; the bucket histogram is additive, so the
    // histogram of chunk i runs while chunk i+1 is still on the PCIe bus.
    ColPtrs c{};
    const bool host_input = hc.mem != TAD_MEM_DEVICE && R > 0;
    PipeShape shape;
    shape.rows = R;
    shape.host = host_input ? &hc : nullptr;
    shape.algo = sp.algo;
    shape.resume = job->share != 0;
    PipeSizes z = pipe_sizes(shape);
    for (int i = 0; i < 10; i++) {
        void *src = col_ptr(hc, i);
        if (!src || R == 0) continue;
        if (hc.mem != TAD_MEM_DEVICE) ensure(ctx, ctx->d_col[i], z.col[i]);
        set_col(c, i, hc.mem == TAD_MEM_DEVICE ? src : ctx->d_col[i].p);
    }
    int nchunks = 1;
    if (host_input) {
        nchunks = (int)((R + (8u << 20) - 1) / (8u << 20));          // ~8M rows (232 MB) per chunk
        if (nchunks > kMaxChunks) nchunks = kMaxChunks;
        if (nchunks < 1) nchunks = 1;
    }
    auto chunk_lo = [&](int k) -> uint64_t {      // host chunk k is [chunk_lo(k), chunk_lo(k + 1)): 16-byte aligned columns
        return k == 0 ? 0 : k == nchunks ? R : std::min<uint64_t>(((R * (uint64_t)k / nchunks) + 15) & ~uint64_t(15), R);
    };
    mark(-1);
    if (host_input) {
        CU(cudaEventRecord(ctx->start_ev, st));
        CU(cudaStreamWaitEvent(ctx->copy_stream, ctx->start_ev, 0));   // workspace of the previous job is free
        for (int k = 0; k < nchunks; k++) {
            const uint64_t lo = chunk_lo(k), hi = chunk_lo(k + 1);
            for (int i = 0; i < 10 && hi > lo; i++) {
                const char *src = static_cast<const char *>(col_ptr(hc, i));
                if (!src) continue;
                const size_t w = col_bytes(i, 1);
                CU(cudaMemcpyAsync(static_cast<char *>(ctx->d_col[i].p) + lo * w, src + lo * w, (hi - lo) * w,
                                   cudaMemcpyHostToDevice, ctx->copy_stream));
            }
            CU(cudaEventRecord(ctx->chunk_ev[k], ctx->copy_stream));
        }
    }

    const RowFilter f = filters ? row_filter(ctx, job, c.src_ns || c.dst_ns) : RowFilter{};
    // launch(cols, rows) over the input: host input once per non-empty chunk, each behind its copy (the copies and the
    // overlapped launches are the H2D phase); device input in one launch that closes `phase`
    auto feed_chunks = [&](auto launch, int phase) {
        mark(-1);
        if (host_input) {
            for (int k = 0; k < nchunks; k++) {
                const uint64_t lo = chunk_lo(k), hi = chunk_lo(k + 1);
                CU(cudaStreamWaitEvent(st, ctx->chunk_ev[k], 0));
                if (hi <= lo) continue;
                CU(launch(offset_cols(c, lo), hi - lo)); launches++;
            }
            mark(TAD_PHASE_H2D);
        } else {
            CU(launch(c, R)); launches += R ? 1 : 0;
            mark(phase);
        }
    };

    // ---- partition -------------------------------------------------------------------------
    const int world = ctx->cfg.world_size, me = ctx->cfg.rank;
    uint64_t R_total = R;
    ensure(ctx, ctx->small, tad_ctx::kSmallDevWords * 8);
    unsigned long long *d_small = static_cast<unsigned long long *>(ctx->small.p);
    if (world > 1 && pass) {
        R_total = pass->global_rows;   // the pass's total from the all-gathered counts
    } else if (world > 1 && sp.global_rows) {
        R_total = sp.global_rows;      // the host counted the table: no start-of-job collective, no host sync
    } else if (world > 1) {
        // global row count -> same bucket count on every rank
        ctx->h_small[0] = R;
        gather_small(ctx, 1, false);
        mark(TAD_PHASE_SYNC);          // arrival skew of the ranks at job start (avoided when the host passes global_rows)
        R_total = 0;
        for (int r = 0; r < world; r++) R_total += ctx->h_small[1 + r];
    }
    const uint32_t B = buckets(ctx, R_total);      // global buckets
    const int logB = __builtin_ctz(B);
    const uint32_t Bl = B >> log_world(ctx);       // buckets owned by one rank
    const uint32_t b_lo = Bl * (uint32_t)me;
    constexpr uint32_t kSlot = kGroupCap;      // = the largest shared-memory class: overflow is as rare as a spill was
    shape.B = B;
    shape.Bl = Bl;
    shape.optimistic = world == 1 && one_gpu_optimistic(ctx, R, B) && !force_exact;
    z = pipe_sizes(shape);
    ensure(ctx, ctx->hist, z.hist);
    ensure(ctx, ctx->offsets, z.offsets);
    ensure(ctx, ctx->cursor, z.cursor);
    ensure(ctx, ctx->big_list, z.big_list);
    ensure(ctx, ctx->big_base, z.big_base);
    ensure(ctx, ctx->cls_list, z.cls_list);
    ensure(ctx, ctx->nsb, z.nsb);
    ensure(ctx, ctx->npb, z.npb);
    // part[] (exact partition: 32 B per local row) is not needed when the multi-GPU optimistic path runs out of the exported
    // slot buffer; the exact multi-GPU branch allocates it on demand
    if (world == 1) ensure(ctx, ctx->part, z.part);
    uint32_t *hist = (uint32_t *)ctx->hist.p, *offsets = (uint32_t *)ctx->offsets.p, *cursor = (uint32_t *)ctx->cursor.p;
    uint32_t *big_base = (uint32_t *)ctx->big_base.p;
    uint32_t *cls_list = (uint32_t *)ctx->cls_list.p;
    uint32_t *big_list = (uint32_t *)ctx->big_list.p, *nsb = (uint32_t *)ctx->nsb.p, *npb = (uint32_t *)ctx->npb.p;
    Row32 *part = (Row32 *)ctx->part.p;

    CU(cudaMemsetAsync(nsb, 0, (size_t)Bl * 4, st));
    CU(cudaMemsetAsync(npb, 0, (size_t)Bl * 4, st));
    SegDesc seg{};
    SeriesEntry *entries = nullptr;
    uint64_t kept = 0, owned = 0;
    bool partitioned = false;
    uint32_t n_ovf = 0;
    const Row32 *ovf_rows = nullptr;
    // ---- single GPU, optimistic partition: no histogram pass.  Bucket b owns a fixed slot of kGroupCap rows; a
    // row that finds its slot full goes to the overflow list, and such buckets take the spill path.  With host input
    // the scatter of H2D chunk i runs while chunk i+1 is on the bus.  Falls back to the exact two-pass partition
    // when the overflow list fills up (heavily skewed tables).
    if (shape.optimistic) {
        const uint64_t ovf_cap = z.ovf / sizeof(Row32);
        ensure(ctx, ctx->part, z.slots);
        ensure(ctx, ctx->ovf, z.ovf);
        part = (Row32 *)ctx->part.p;
        Row32 *ovf = (Row32 *)ctx->ovf.p;
        CU(cudaMemsetAsync(cursor, 0, (size_t)B * 4, st));
        feed_chunks([&](const ColPtrs &cc, uint64_t n) {
            return launch_scatter(st, cc, n, f, logB, cursor, part, kSlot, ovf, (uint32_t)ovf_cap, d_stats + ST_OVF);
        }, TAD_PHASE_SCATTER);
        // arrival counts -> (virtual) bucket offsets, capacity-class lists, list of over-full buckets
        CU(launch_bucket_scan(st, cursor, offsets, hist /* unused cursor copy */, B, kSlot, big_list, big_base, cls_list,
                              d_stats, ctx->scan_sync.p, ++ctx->scan_epoch)); launches++;
        mark(TAD_PHASE_SCAN);
        read_stats();
        if (ctx->h_stats[ST_OVF] <= ovf_cap) {
            partitioned = true;
            n_ovf = ctx->h_stats[ST_OVF];
            ovf_rows = ovf;
            kept = owned = ctx->h_stats[ST_KEPT];
            seg.nseg = 1;
            seg.base[0] = part;
            seg.off[0] = offsets;
            seg.stride = kSlot;
            shape.owned = owned;
            ensure(ctx, ctx->entries, pipe_sizes(shape).entries);
            entries = static_cast<SeriesEntry *>(ctx->entries.p);
        } else {
            CU(cudaMemsetAsync(d_stats, 0, 64 * sizeof(uint32_t), st));      // discard; redo exactly
        }
    }

    // ---- exported buffer + peer mappings (multi-GPU peer pull) -----------------------------------------------------------
    // blocking 128-byte all-gathers (rare: regrow, exact-path row counts): rank r's words land at h_small + G * (1 + r)
    constexpr int G = tad_ctx::kGatherMax;
    // Every rank calls this with the SAME `need` in the same job (it depends only on values all ranks share), so all ranks
    // regrow together: unmap, barrier (nobody maps a buffer that is about to be freed), reallocate, exchange the IPC
    // handles, map.  First job or a larger table only.
    auto ensure_exported = [&](size_t need) {
        // the decision must be the same on every rank: it is taken on the size the ranks last agreed on, not on the local
        // capacity (which may differ when one rank's allocation fell back to the exact size under memory pressure)
        if (need <= ctx->x_agreed && ctx->peers_mapped) return;
        CU(unmap_peers(ctx));
        memset(ctx->h_small, 0, G * 8);
        gather_small(ctx, G, false);
        ensure(ctx, ctx->xbuf, need);
        memset(ctx->h_small, 0, G * 8);
        ctx->h_small[0] = ctx->xbuf.cap;
        CU(nccl_ipc_export(&ctx->nccl, ctx->xbuf.p, ctx->h_small + 2));      // a 64-byte handle in words 2..9
        gather_small(ctx, G, false);
        for (int r = 0; r < world; r++) {
            if (r == me) continue;
            if (ctx->h_small[G * (1 + r)] < need) fail(TAD_ERR_INTERNAL, "rank %d exports a smaller partition buffer", r);
            cudaError_t e = nccl_ipc_map(&ctx->nccl, ctx->h_small + G * (1 + r) + 2, &ctx->peer_x[r]);
            if (e != cudaSuccess) {
                cudaGetLastError();
                ctx->peer_x[r] = nullptr;
                fail(TAD_ERR_CUDA, "cannot map the partition buffer of rank %d (%s); set TAD_PEER_PULL=0 on every rank to "
                                   "exchange rows through NCCL instead", r, cudaGetErrorString(e));
            }
        }
        ctx->peers_mapped = true;
        ctx->x_agreed = need;
    };
    // ---- several GPUs, optimistic partition + peer pull ---------------------------------------------------------------
    // Every rank scatters its rows into fixed-capacity slots of ALL global buckets (slot = kGroupCap / world rows: a
    // source holds 1/world of a bucket on average) inside a buffer its peers have mapped with CUDA IPC.  One 8-byte
    // all-gather after the scatter is the barrier "every rank's slots are complete" and carries the overflow counts: if
    // any slot overflowed anywhere, all ranks take the exact path below (same decision everywhere: it is made on the
    // gathered data).  Otherwise each rank reads the arrival counters of its bucket range out of the peers' buffers and
    // its group kernel pulls the rows themselves, segment by segment, with the bulk copies it issues anyway.
    const uint32_t slotM = slot(ctx);
    const size_t x_cnt_bytes = xbuf_cnt_bytes(B);
    // the peers' exported partitions as segments: rank r's rows from skip[r] (null: 0), its offsets at off + r * off_stride
    auto peer_segments = [&](const uint32_t *off, size_t off_stride, const unsigned long long *skip) {
        seg.nseg = world;
        for (int r = 0; r < world; r++) {
            const char *xb = r == me ? static_cast<const char *>(ctx->xbuf.p) : static_cast<const char *>(ctx->peer_x[r]);
            seg.base[r] = reinterpret_cast<const Row32 *>(xb + x_cnt_bytes) + (skip ? skip[r] : 0);
            seg.off[r] = off + r * off_stride;
        }
    };
    if (world > 1 && slots_allowed(ctx, R_total) && !force_exact) {
        ensure_exported(slot_xbuf_bytes(ctx, B));
        uint32_t *xcursor = static_cast<uint32_t *>(ctx->xbuf.p);
        Row32 *xpart = reinterpret_cast<Row32 *>(static_cast<char *>(ctx->xbuf.p) + x_cnt_bytes);
        ensure(ctx, ctx->xcnt, (size_t)Bl * 4 * world);
        ensure(ctx, ctx->xtotal, (size_t)Bl * 4);
        uint32_t *xcnt = (uint32_t *)ctx->xcnt.p, *xtotal = (uint32_t *)ctx->xtotal.p;
        CU(cudaMemsetAsync(xcursor, 0, (size_t)B * 4, st));
        feed_chunks([&](const ColPtrs &cc, uint64_t n) {
            return launch_scatter(st, cc, n, f, logB, xcursor, xpart, slotM, nullptr, 0, d_stats + ST_OVF);
        }, TAD_PHASE_SCATTER);
        // barrier + overflow agreement: {overflow rows, -} of every rank
        if (nccl_allgather(&ctx->nccl, d_stats + ST_OVF, d_small + tad_ctx::kWOvf, 8, st))
            fail(TAD_ERR_NCCL, "%s", nccl_last_error());
        mark(TAD_PHASE_SYNC);
        PeerCounters pc{};
        for (int r = 0; r < world; r++) pc.p[r] = r == me ? xcursor : static_cast<const uint32_t *>(ctx->peer_x[r]);
        CU(launch_gather_counts(st, pc, world, b_lo, Bl, slotM, xcnt, xtotal, xcursor, B, d_stats + ST_LOCALKEPT)); launches += 2;
        mark(TAD_PHASE_EXCHANGE);
        CU(launch_bucket_scan(st, xtotal, offsets, cursor, Bl, kGroupCap, big_list, big_base, cls_list, d_stats,
                              ctx->scan_sync.p, ++ctx->scan_epoch)); launches++;
        mark(TAD_PHASE_SCAN);
        CU(cudaMemcpyAsync(ctx->h_small + tad_ctx::kWOvf, d_small + tad_ctx::kWOvf, 8 * world, cudaMemcpyDeviceToHost, st));
        read_stats();
        check_cancel();
        uint64_t any_ovf = 0;
        for (int r = 0; r < world; r++) any_ovf += (uint32_t)ctx->h_small[tad_ctx::kWOvf + r];
        if (any_ovf == 0) {
            partitioned = true;
            kept = ctx->h_stats[ST_LOCALKEPT];
            owned = ctx->h_stats[ST_KEPT];
            seg.stride = slotM;
            seg.b_lo = b_lo;
            peer_segments(xcnt, Bl, nullptr);
            ensure(ctx, ctx->entries, (owned ? owned : 1) * sizeof(SeriesEntry));
            entries = static_cast<SeriesEntry *>(ctx->entries.p);
        } else {
            CU(cudaMemsetAsync(d_stats, 0, 64 * sizeof(uint32_t), st));      // discard; redo exactly (every rank does)
        }
    }
    if (world == 1 && !partitioned) {
        CU(cudaMemsetAsync(hist, 0, (size_t)B * 4, st));
        feed_chunks([&](const ColPtrs &cc, uint64_t n) { return launch_hist(st, cc, n, f, logB, hist); }, TAD_PHASE_HIST);
        // single GPU: these are the final bucket offsets; multi GPU: offsets inside the local send buffer
        CU(launch_bucket_scan(st, hist, offsets, cursor, B, world > 1 ? 0xffffffffu : (uint32_t)kGroupCap, big_list, big_base,
                              world > 1 ? nullptr : cls_list, d_stats, ctx->scan_sync.p, ++ctx->scan_epoch)); launches++;
        mark(TAD_PHASE_SCAN);
        CU(launch_scatter(st, c, R, f, logB, cursor, part)); launches += R ? 1 : 0;
        mark(TAD_PHASE_SCATTER);
        read_stats();
        kept = owned = ctx->h_stats[ST_KEPT];
        seg.nseg = 1;
        seg.base[0] = part;
        seg.off[0] = offsets;
        entries = reinterpret_cast<SeriesEntry *>(part);      // in place over the staged bucket rows
    } else if (world > 1 && !partitioned) {
        // ---- multi GPU, exact partition: K row chunks; chunk c is sent over NVLink (comm stream) while chunk c+1 is scattered ------
        // chunked (overlapped) exchange pays off at N = 2 (measured 11.5 -> 9.6 ms); at N >= 4 the NVLink all-to-all is
        // longer than the scatter it could hide behind and the extra segments cost the group kernel more than is won
        // With peer pull (default) the exact partition is written into the EXPORTED buffer and the owners' group kernels read
        // their segments straight out of the peers' copies: no receive buffer, no all-to-all (and no chunking: K = 1).
        const bool pull = ctx->peer_pull != 0 && ctx->exact_pull != 0;
        const uint64_t k_rows = pass ? pass->max_rows : R;      // a pass: the same chunk count on every rank
        const int K = pull ? 1 : (k_rows >= ctx->exchange_min_rows && (world == 2 || ctx->exchange_chunks_forced)) ? ctx->exchange_chunks : 1;
        auto xlo = [&](int cidx) -> uint64_t {
            if (cidx <= 0) return 0;
            if (cidx >= K) return R;
            const uint64_t v = ((R * (uint64_t)cidx / K) + 15) & ~uint64_t(15);
            return v < R ? v : R;
        };
        const int NS = world * K;                              // segments: (source rank, chunk)
        if (pull) {
            // the exported buffer must hold the largest shard: the ranks agree on it (blocking 128-byte all-gather; this path
            // is the fallback for skewed or very large tables, where a host sync more does not matter)
            memset(ctx->h_small, 0, G * 8);
            ctx->h_small[0] = R;
            gather_small(ctx, G, false);
            uint64_t max_rows = 0;
            for (int r = 0; r < world; r++) max_rows = std::max<uint64_t>(max_rows, ctx->h_small[G * (1 + r)]);
            ensure_exported(xbuf_bytes(ctx, R_total, max_rows, false));
            part = reinterpret_cast<Row32 *>(static_cast<char *>(ctx->xbuf.p) + x_cnt_bytes);
        } else {
            ensure(ctx, ctx->part, (R ? R : 1) * sizeof(Row32));
            part = (Row32 *)ctx->part.p;
        }
        for (const auto &b : exact_bufs(ctx, B, Bl, K)) ensure(ctx, *b.first, b.second);
        hist = (uint32_t *)ctx->hist.p; offsets = (uint32_t *)ctx->offsets.p; cursor = (uint32_t *)ctx->cursor.p;
        uint32_t *hist_all = (uint32_t *)ctx->hist_all.p, *seg_off = (uint32_t *)ctx->seg_off.p;
        uint32_t *seg_total = (uint32_t *)ctx->seg_total.p;
        CU(cudaMemsetAsync(hist, 0, (size_t)B * 4 * K, st));
        if (host_input)
            for (int k = 0; k < nchunks; k++) CU(cudaStreamWaitEvent(st, ctx->chunk_ev[k], 0));
        mark(TAD_PHASE_H2D);
        for (int cx = 0; cx < K; cx++) {
            const uint64_t lo = xlo(cx), hi = xlo(cx + 1);
            if (hi > lo) { CU(launch_hist(st, offset_cols(c, lo), hi - lo, f, logB, hist + (size_t)cx * B)); launches++; }
        }
        mark(TAD_PHASE_HIST);
        for (int cx = 0; cx < K; cx++) {
            CU(launch_bucket_scan(st, hist + (size_t)cx * B, offsets + (size_t)cx * (B + 1), cursor + (size_t)cx * B, B, 0xffffffffu,
                                  big_list, big_base, nullptr, d_stats, ctx->scan_sync.p, ++ctx->scan_epoch)); launches++;
        }
        mark(TAD_PHASE_SCAN);
        // every rank learns every (rank, chunk) histogram: segment offsets of the owned bucket range, receive sizes
        if (nccl_allgather(&ctx->nccl, hist, hist_all, (size_t)B * 4 * K, st)) fail(TAD_ERR_NCCL, "%s", nccl_last_error());
        unsigned long long *pull_skip = ctx->h_small + tad_ctx::kWPullSkip;
        CU(launch_segment_scan(st, hist_all, B, b_lo, Bl, NS, seg_off, seg_total, d_small,
                               pull ? d_small + tad_ctx::kWPullSkip : nullptr)); launches += 2;
        CU(cudaMemcpyAsync(ctx->h_small, d_small, 8 * NS, cudaMemcpyDeviceToHost, st));
        if (pull) CU(cudaMemcpyAsync(pull_skip, d_small + tad_ctx::kWPullSkip, 8 * NS, cudaMemcpyDeviceToHost, st));
        for (int cx = 0; cx < K; cx++)        // send boundaries of chunk cx: offsets_cx[p * Bl], p = 0..world
            CU(cudaMemcpy2DAsync(ctx->h_small + tad_ctx::kWSendLo + cx * (kMaxRanks + 1), 8, offsets + (size_t)cx * (B + 1),
                                 (size_t)Bl * 4, 4, world + 1, cudaMemcpyDeviceToHost, st));
        CU(cudaStreamSynchronize(st));
        check_cancel();
        uint64_t recv_off[kMaxSeg], recv_total = 0, send_lo[kMaxXChunks][kMaxRanks + 1];
        for (int sgi = 0; sgi < NS; sgi++) {
            recv_off[sgi] = recv_total;
            if (sgi / K != me) recv_total += ctx->h_small[sgi] * 32;
            owned += ctx->h_small[sgi];
        }
        for (int cx = 0; cx < K; cx++) {
            for (int p = 0; p <= world; p++)
                send_lo[cx][p] = (uint32_t)ctx->h_small[tad_ctx::kWSendLo + cx * (kMaxRanks + 1) + p];
            kept += send_lo[cx][world];
        }
        if (owned >= (1ull << 32) - 1) fail(TAD_ERR_INVALID_ARG, "more than 2^32-2 rows owned by one GPU after the exchange");
        cudaStream_t cs = ctx->copy_stream;
        if (pull) {
            CU(launch_scatter(st, c, R, f, logB, cursor, part)); launches += R ? 1 : 0;
            mark(TAD_PHASE_SCATTER);
            // barrier: every rank's exact partition is complete
            if (peer_barrier(ctx)) fail(TAD_ERR_NCCL, "%s", nccl_last_error());
            mark(TAD_PHASE_SYNC);
            peer_segments(seg_off, Bl + 1, pull_skip);      // rows in front of my range skipped
        } else {
            ensure(ctx, ctx->exch, recv_total ? recv_total : 32);
            for (int cx = 0; cx < K; cx++) {
                const uint64_t lo = xlo(cx), hi = xlo(cx + 1);
                if (hi > lo) { CU(launch_scatter(st, offset_cols(c, lo), hi - lo, f, logB, cursor + (size_t)cx * B, part + lo)); launches++; }
                CU(cudaEventRecord(ctx->x_ev[cx], st));
                CU(cudaStreamWaitEvent(cs, ctx->x_ev[cx], 0));
                uint64_t so[kMaxRanks], sb[kMaxRanks], ro[kMaxRanks], rb[kMaxRanks];
                for (int p = 0; p < world; p++) {
                    so[p] = (lo + send_lo[cx][p]) * 32;
                    sb[p] = (send_lo[cx][p + 1] - send_lo[cx][p]) * 32;
                    ro[p] = recv_off[p * K + cx];
                    rb[p] = ctx->h_small[p * K + cx] * 32;
                }
                if (nccl_alltoallv(&ctx->nccl, part, so, sb, ctx->exch.p, ro, rb, cs)) fail(TAD_ERR_NCCL, "%s", nccl_last_error());
            }
            mark(TAD_PHASE_SCATTER);
            CU(cudaEventRecord(ctx->x_ev[K], cs));
            CU(cudaStreamWaitEvent(st, ctx->x_ev[K], 0));
            seg.nseg = NS;
            for (int sgi = 0; sgi < NS; sgi++) {
                const int r = sgi / K, cx = sgi % K;
                seg.base[sgi] = r == me ? part + xlo(cx) + send_lo[cx][me]
                                        : reinterpret_cast<const Row32 *>((const char *)ctx->exch.p + recv_off[sgi]);
                seg.off[sgi] = seg_off + (size_t)sgi * (Bl + 1);
            }
        }
        // final (virtual) bucket offsets of the owned range, oversized-bucket list, capacity-class lists
        CU(launch_bucket_scan(st, seg_total, offsets, cursor, Bl, kGroupCap, big_list, big_base, cls_list, d_stats,
                              ctx->scan_sync.p, ++ctx->scan_epoch)); launches++;
        mark(TAD_PHASE_EXCHANGE);           // = the part of the exchange NOT hidden behind the scatter
        read_stats();
        ensure(ctx, ctx->entries, (owned ? owned : 1) * sizeof(SeriesEntry));
        entries = static_cast<SeriesEntry *>(ctx->entries.p);
    }
    check_cancel();
    const uint32_t n_big = ctx->h_stats[ST_NBIG];
    const uint64_t big_rows = ctx->h_stats[ST_BIGROWS];
    set_progress(job, TAD_STATE_RUNNING, 3);    // ingest, partition, exchange

    // ---- group ------------------------------------------------------------------------------
    shape.owned = owned;
    z = pipe_sizes(shape);
    ensure(ctx, ctx->csr_v, z.csr_v);
    ensure(ctx, ctx->csr_t, z.csr_t);
    uint64_t *csr_v = (uint64_t *)ctx->csr_v.p;
    uint32_t *csr_t = (uint32_t *)ctx->csr_t.p;
    uint32_t *csr_p = nullptr;
    if (sp.algo == TAD_ALGO_DBSCAN) {
        ensure(ctx, ctx->csr_p, z.csr_p);
        csr_p = (uint32_t *)ctx->csr_p.p;
    }
    // EWMA is scored inside the group kernel (launch_group_ewma, in the detect loop below): only the spilled buckets go
    // through the per-series arrays, the series scan and the detect kernel
    const bool fused = sp.algo == TAD_ALGO_EWMA;
    uint32_t n_cls[kGroupClasses];                        // buckets of every capacity class
    std::copy(ctx->h_stats + ST_NCLS0, ctx->h_stats + ST_NCLS0 + kGroupClasses, n_cls);
    mark(-1);
    {
        int l = 0;
        if (ctx->sort_classes) {
            // class lists in ascending bucket order: concurrently running CTAs then touch neighbouring slots / csr stretches
            const size_t need = sort_lists_scratch_bytes(Bl);
            ensure(ctx, ctx->sortb, need);
            int bits = 1;
            while ((1u << bits) < Bl && bits < 32) bits++;
            for (int k = 0; k < kGroupClasses; k++)
                if (n_cls[k] > 1) { CU(sort_bucket_list(st, cls_list + (size_t)k * Bl, n_cls[k], bits, ctx->sortb.p, ctx->sortb.cap)); launches += 3; }
        }
        if (!fused) {
            CU(launch_group(st, seg, entries, offsets, Bl, cls_list, n_cls, csr_v, csr_t, csr_p, nsb, npb, sp.reducer, &l));
            launches += l;
        }
    }
    mark(TAD_PHASE_GROUP);
    if (n_big) {
        const size_t need = spill_scratch_bytes(big_rows);
        if (!fits(ctx, ctx->spill, need)) throw PassSplit{"oversized-bucket scratch", need, ctx->held};
        ensure(ctx, ctx->spill, need);
        int l = 0;
        CU(run_spill(st, seg, entries, offsets, big_list, big_base, n_big, big_rows, ctx->spill.p, ctx->spill.cap, csr_v, csr_t,
                     nsb, npb, sp.reducer, &l, ovf_rows, n_ovf));
        launches += l;
        mark(TAD_PHASE_SPILL);
    }
    ensure(ctx, ctx->sbase, z.sbase);      // series base per bucket + bucket hint per 32 series
    uint32_t *sbase = (uint32_t *)ctx->sbase.p;
    uint32_t S = 0;                        // series of the detect kernels (EWMA: of the spilled buckets)
    uint64_t points = 0;
    if (!fused || n_big) {
        CU(launch_series_scan(st, nsb, npb, sbase, Bl, d_stats, ctx->scan_sync.p, ++ctx->scan_epoch)); launches++;
        read_stats();
        check_cancel();
        S = ctx->h_stats[ST_SERIES];
        points = ctx->h_stats[ST_POINTS];
    }
    if (!fused) set_progress(job, TAD_STATE_RUNNING, 4);

    // ---- detect -----------------------------------------------------------------------------
    const bool emit_all = (sp.flags & TAD_FLAG_EMIT_ALL) != 0;
    // EWMA: the points are counted by the scoring kernel itself, so the first guess comes from the rows
    uint64_t out_cap = out_cap_guess(fused ? owned : points, emit_all);
    uint64_t out_rows = 0;
    OutLayout L{};
    OutCols oc{};
    shape.series = S;
    double parked_ms = 0;                 // the ARIMA fit's time parked while other jobs ran: not this job's device time
    for (int attempt = 0; attempt < 3; attempt++) {
        shape.out_cap = out_cap;
        z = pipe_sizes(shape);
        L = out_layout(out_cap);
        if (!fits(ctx, ctx->outb, z.outb)) throw PassSplit{"result buffer", z.outb, ctx->held};
        ensure(ctx, ctx->outb, z.outb);
        oc = out_cols(ctx->outb.p, L);
        CU(cudaMemsetAsync(d_stats + ST_OUTCOUNT, 0, 4, st));
        mark(-1);
        if (fused) {
            // the group kernel never writes over the rows it reads: a rerun with larger capacity scores them again
            CU(cudaMemsetAsync(d_stats + ST_GSERIES, 0, 8, st));
            int l = 0;
            CU(launch_group_ewma(st, seg, offsets, Bl, cls_list, n_cls, sp.reducer,
                                 GroupScore{oc, (uint32_t)out_cap, d_stats, emit_all}, &l));
            launches += l;
            mark(TAD_PHASE_GROUP);
            CU(launch_detect_ewma(st, entries, offsets, sbase, Bl, S, csr_v, csr_t, oc, (uint32_t)out_cap, d_stats, emit_all));
            launches += S ? 1 : 0;
        } else if (sp.algo == TAD_ALGO_DBSCAN) {
            ensure(ctx, ctx->dbx, z.dbx);         // prefix count of core points, per point slot
            ensure(ctx, ctx->dbi, z.dbi);         // noise flag, per point slot
            CU(launch_detect_dbscan(st, entries, offsets, sbase, Bl, S, csr_v, csr_t, csr_p, (uint32_t *)ctx->dbx.p,
                                    (uint8_t *)ctx->dbi.p, oc, (uint32_t)out_cap, d_stats, emit_all));
            launches += S ? 1 : 0;
        } else if (sp.algo == TAD_ALGO_ARIMA) {
            ensure(ctx, ctx->ar_y, z.ar_y);
            ensure(ctx, ctx->ar_pred, z.ar_pred);
            ensure(ctx, ctx->ar_lam, z.ar_lam);
            ensure(ctx, ctx->ar_res, z.ar_res);
            if (attempt == 0 && S) {
                uint32_t *res = job->share ? (uint32_t *)ctx->ar_res.p : nullptr;
                CU(cudaMemsetAsync(d_stats + ST_FITS, 0, 12, st));      // fit counters and cancel word
                if (res) CU(cudaMemsetAsync(res + 2 * (size_t)S, 0, 8, st));
                // this pass's fit, also the part a job run in its yield may fit beside (its buffers stay parked meanwhile)
                const tad_progress before = progress_of(job);
                YieldedFit fit{job,
                               FitPart{entries, offsets, sbase, Bl, S, (double *)ctx->ar_y.p, (double *)ctx->ar_lam.p,
                                       (double *)ctx->ar_pred.p, d_stats + ST_FITS + 2, d_stats + ST_FITS + 1, res,
                                       d_stats + ST_FITS},
                               before.fits_done, before.fits_total};
                if (ctx->beside && ctx->beside->job != job)        // this job runs in that yield: it fits beside it
                    parked_ms = fit_beside(ctx, fit, *ctx->beside, csr_v, d_stats + ST_FITS + 3, launches);
                else
                    parked_ms = fit_solo(ctx, fit, csr_v, launches);
                // pred[] is incomplete: no detect.  Several GPUs: the rank goes on to the verdict, which fails the job
                check_cancel();
                const tad_ctx::FitCounts &end = ctx->h_fit->part[0].end;
                if (world > 1 && end.done < end.total) out.fit_stop = board_stopper(ctx, job);
            }
            if (out.fit_stop < 0) {
                CU(launch_detect_arima(st, entries, offsets, sbase, Bl, S, csr_v, csr_t, (const double *)ctx->ar_pred.p,
                                       (const double *)ctx->ar_lam.p, oc, (uint32_t)out_cap, d_stats, emit_all));
                launches += S ? 1 : 0;
            }
        } else {
            fail(TAD_ERR_UNSUPPORTED, "algorithm %d is not implemented by this build", sp.algo);
        }
        mark(TAD_PHASE_DETECT);
        read_stats();
        out_rows = ctx->h_stats[ST_OUTCOUNT];
        if (out_rows <= out_cap) break;
        out_cap = out_rows;                 // capacity guess too small: rerun detect (idempotent)
        if (attempt == 2) fail(TAD_ERR_INTERNAL, "result capacity did not converge");
    }
    check_cancel();
    uint64_t series_all = S, points_all = points;
    if (fused) {
        series_all += ctx->h_stats[ST_GSERIES];
        points_all += ctx->h_stats[ST_GPOINTS];
        set_progress(job, TAD_STATE_RUNNING, 4);
    }
    set_progress(job, TAD_STATE_RUNNING, 5);
    if (world > 1 && !pass) {
        // the verdict: an 8-byte all-gather of every rank's stop_word, on which every rank fails or goes on alike, so a
        // cancel on one rank never leaves a peer waiting in a collective.  It is also the end-of-job barrier of the
        // peer-pull paths: my slots and counters may be overwritten (next job) only after every peer's group kernel has
        // read them.  Its wait is the ranks' arrival skew, accounted as TAD_PHASE_SYNC.
        mark(-1);
        ctx->h_small[tad_ctx::kWBarrier] = stop_word(job, out.fit_stop);
        CU(cudaMemcpyAsync(d_small + tad_ctx::kWBarrier, ctx->h_small + tad_ctx::kWBarrier, 8, cudaMemcpyHostToDevice, st));
        if (peer_barrier(ctx)) fail(TAD_ERR_NCCL, "%s", nccl_last_error());
        mark(TAD_PHASE_SYNC);
        CU(cudaMemcpyAsync(ctx->h_small + tad_ctx::kWBarrierIn, d_small + tad_ctx::kWBarrierIn, 8 * world,
                           cudaMemcpyDeviceToHost, st));
        CU(cudaStreamSynchronize(st));
        agree_stop(ctx->h_small + tad_ctx::kWBarrierIn, world);
    }

    // ---- egress: result rows -> pinned host memory -------------------------------------------
    mark(-1);
    {
        OutLayout HL = out_layout(out_rows ? out_rows : 1);
        out.block = take_pinned(ctx, HL.total);
        char *hb = static_cast<char *>(out.block.p);
        const char *db = static_cast<const char *>(ctx->outb.p);
        for (int i = 0; i < 11 && out_rows; i++)
            CU(cudaMemcpyAsync(hb + HL.off[i], db + L.off[i], kOutWidth[i] * out_rows, cudaMemcpyDeviceToHost, st));
    }
    mark(TAD_PHASE_D2H);
    CU(cudaStreamSynchronize(st));

    // ---- status ---------------------------------------------------------------------------------
    double phase_ms[TAD_NPHASES] = {0};
    float total = 0;
    for (int i = 1; i < nev; i++) {
        if (ev_phase[i] < 0) continue;
        float ms = 0;
        CU(cudaEventElapsedTime(&ms, ctx->ev[i - 1], ctx->ev[i]));
        phase_ms[ev_phase[i]] += ms;
    }
    // device span excludes the H2D/D2H copies: first partition event .. last detect event
    int first_k = -1, last_k = -1;
    for (int i = 0; i < nev; i++) {
        if ((ev_phase[i] == TAD_PHASE_HIST || ev_phase[i] == TAD_PHASE_H2D || ev_phase[i] == TAD_PHASE_SCATTER) && first_k < 0)
            first_k = i - 1;
        if (ev_phase[i] == TAD_PHASE_DETECT || (ev_phase[i] == TAD_PHASE_SYNC && last_k >= 0)) last_k = i;
    }
    if (first_k >= 0 && last_k > first_k) CU(cudaEventElapsedTime(&total, ctx->ev[first_k], ctx->ev[last_k]));
    if (parked_ms > 0) {
        phase_ms[TAD_PHASE_DETECT] = std::max(0.0, phase_ms[TAD_PHASE_DETECT] - parked_ms);
        total = (float)std::max(0.0, (double)total - parked_ms);
    }
    out.kept = kept;
    out.owned = owned;
    out.points = points_all;
    out.series = series_all;
    out.out_rows = out_rows;
    out.spill_rows = big_rows;
    out.launches = launches;
    out.device_ms = total;
    for (int i = 0; i < TAD_NPHASES; i++) out.phase_ms[i] = phase_ms[i];
}
void publish_rows(tad_job *job, PinnedBlock block, uint64_t rows)
{
    job->result_block = block;
    OutCols ho = out_cols(block.p, out_layout(rows ? rows : 1));
    job->rows.rows = rows;
    job->rows.src_ip = ho.src_ip; job->rows.dst_ip = ho.dst_ip;
    job->rows.src_port = ho.src_port; job->rows.dst_port = ho.dst_port;
    job->rows.proto = ho.proto; job->rows.flow_start = ho.flow_start; job->rows.flow_end = ho.flow_end;
    job->rows.stddev = ho.stddev; job->rows.algo_calc = ho.algo_calc; job->rows.throughput = ho.throughput;
    job->rows.anomaly = ho.anomaly;
}

// The single-GPU pipeline's shape for `rows` input rows, with upper bounds for the rows owned, series and points; the
// optimistic partition where asked for and its slot buffer may be used.
PipeShape one_gpu_shape(const tad_ctx *ctx, const tad_job *job, uint64_t rows, bool optimistic)
{
    PipeShape s;
    s.rows = rows;
    s.algo = job->spec.algo;
    s.B = s.Bl = buckets(ctx, rows);
    s.optimistic = optimistic && one_gpu_optimistic(ctx, rows, s.B);
    s.resume = job->share != 0;
    s.owned = s.series = rows;
    s.out_cap = out_cap_guess(rows, (job->spec.flags & TAD_FLAG_EMIT_ALL) != 0);
    return s;
}

// Workspace of one pass of `rows` rows: the pipeline over device columns, the pass's key/value columns (d_col[0..7],
// `col_rows` rows each), the host chunk staging and the pass counters.  fresh: on an empty workspace.
size_t pass_need(tad_ctx *ctx, const tad_job *job, uint64_t rows, uint64_t col_rows, bool optimistic, size_t stage_bytes,
                 bool fresh)
{
    PipeSizes z = pipe_sizes(one_gpu_shape(ctx, job, rows, optimistic));
    for (int i = 0; i < 8; i++) z.col[i] = has_col(job, i) ? col_bytes(i, col_rows) : 0;
    auto bufs = pipe_bufs(ctx, z);
    bufs.push_back({&ctx->stage, stage_bytes});
    bufs.push_back({&ctx->pcnt, (kMaxPasses + 1) * 8});
    return workspace_after(ctx, bufs, fresh);
}

// Workspace of a round packed into the host row store, on an empty workspace: the pass columns (`col_rows` rows each),
// the host chunk staging, the pass counters and the out-stage.  The out-stage is freed before the first pass runs, so
// the planner sizes the passes without it and uses the store only where this fits the budget at the planned cap.
size_t store_round_need(tad_ctx *ctx, const tad_job *job, uint64_t col_rows, size_t stage_bytes, size_t ostage_bytes)
{
    std::vector<std::pair<DevBuf *, size_t>> bufs = {{&ctx->stage, stage_bytes}, {&ctx->pcnt, (kMaxPasses + 1) * 8},
                                                     {&ctx->ostage, ostage_bytes}};
    for (int i = 0; i < 8; i++) bufs.push_back({&ctx->d_col[i], has_col(job, i) ? col_bytes(i, col_rows) : 0});
    return workspace_after(ctx, bufs, true);
}

void add_pass(PassOut &acc, const PassOut &o)
{
    acc.kept += o.kept;
    acc.owned += o.owned;
    acc.points += o.points;
    acc.series += o.series;
    acc.out_rows += o.out_rows;
    acc.spill_rows += o.spill_rows;
    acc.launches += o.launches;
    acc.device_ms += o.device_ms;
    for (int i = 0; i < TAD_NPHASES; i++) acc.phase_ms[i] += o.phase_ms[i];
}

// The passes' result rows as one contiguous block, pass after pass (acc.out_rows rows); the passes' blocks go back.
void join_passes(tad_ctx *ctx, std::vector<PassOut> &outs, PassOut &acc)
{
    const OutLayout HL = out_layout(acc.out_rows ? acc.out_rows : 1);
    acc.block = take_pinned(ctx, HL.total);
    uint64_t at = 0;
    for (PassOut &o : outs) {
        const OutLayout PL = out_layout(o.out_rows ? o.out_rows : 1);
        for (int i = 0; i < 11; i++)
            memcpy(static_cast<char *>(acc.block.p) + HL.off[i] + at * kOutWidth[i],
                   static_cast<const char *>(o.block.p) + PL.off[i], kOutWidth[i] * o.out_rows);
        at += o.out_rows;
        give_pinned(ctx, o.block);
        o.block = PinnedBlock{};
    }
}

// ---- streamed input: the worker's side of the hand-over (the caller's side is tad_stream_push / tad_stream_end) ----------
// The next block of the current round; false once the caller has closed the round.  While it waits, a job with
// TAD_FLAG_LEND may lend the GPU to queued jobs (lend).  A rank stream job fails only where its peers fail with it: once
// it is cancelled, its context shuts down or a block was refused, the rest of its round is empty (StreamRound).
bool next_block(tad_job *job, tad_columns &b, tad_text_column *txt)
{
    const double t_wait = now_ms();
    std::unique_lock<std::mutex> lk(job->mu);
    for (;;) {
        if (job->rank_stream && job->ctx->stopping.load()) job->cancel.store(1);
        if (job->rank_stream && (job->cancel.load() || job->peer_stop.load() || job->in.err)) return false;
        if (job->cancel.load()) fail(TAD_ERR_CANCELLED, "job cancelled");
        if (job->ctx->stopping.load()) fail(TAD_ERR_CANCELLED, "context is shutting down");
        if (job->in.err) fail(job->in.err, "%s", job->in.msg);
        if (job->in.has_blk) {
            b = job->in.blk;
            for (int t = 0; t < 4; t++) txt[t] = job->in.txt[t];
            job->in.has_blk = false;
            job->in.taken++;
            job->cv.notify_all();
            return true;
        }
        if (job->in.end_req) return false;
        if (job->lend) {
            lk.unlock();
            lend(job, now_ms() - t_wait);
            lk.lock();
            if (job->in.has_blk || job->in.end_req || job->cancel.load()) continue;
        }
        job->cv.wait_for(lk, std::chrono::milliseconds(5));
    }
}

// The engine no longer reads the first `n` blocks of the job: the pushes waiting for them may return.
void release_blocks(tad_job *job, uint64_t n)
{
    std::lock_guard<std::mutex> lk(job->mu);
    job->in.released = n;
    job->cv.notify_all();
}

// The worker has finished with the round: tad_stream_end returns `again`.
void close_round(tad_job *job, bool again)
{
    std::lock_guard<std::mutex> lk(job->mu);
    job->in.released = job->in.taken;
    job->in.round_start = job->in.taken;
    job->in.end_req = false;
    job->in.again = again;
    job->in.round_done = true;
    job->cv.notify_all();
}

// A streamed job put back in the queue (run_one): the round in progress, if one is, is taken to its end unread and
// closed with again = 1, so that its caller delivers the rows again once the job's turn comes.  A round not yet begun
// is left to that turn: its first block waits there.
void discard_round(tad_job *job)
{
    {
        std::lock_guard<std::mutex> lk(job->mu);
        if (!job->in.end_req && job->in.taken == job->in.round_start) return;
    }
    tad_columns b{};
    tad_text_column tx[4]{};
    while (next_block(job, b, tx)) {
        std::lock_guard<std::mutex> lk(job->mu);
        job->in.released = job->in.taken;
        job->cv.notify_all();
    }
    close_round(job, true);
}

// Device buffer grown to `bytes` with its first `keep` bytes carried over (ensure() frees before it allocates).
void grow_keep(tad_ctx *ctx, DevBuf &b, size_t bytes, size_t keep, cudaStream_t st)
{
    if (bytes <= b.cap) return;
    const DevBuf n = alloc_buf(ctx, bytes);
    if (keep) CU(cudaMemcpyAsync(n.p, b.p, keep, cudaMemcpyDeviceToDevice, st));
    CU(cudaStreamSynchronize(st));
    free_buf(ctx, b);
    b = n;
}

constexpr uint64_t kMaxPassRows = (1ull << 32) - 2;   // the pipeline's offsets are u32: the row cap of one pass

// The largest n <= hi whose workspace need(n) fits `budget`; 0 when none does.
template <class Need>
uint64_t largest_fit(uint64_t hi, uint64_t budget, Need need)
{
    uint64_t lo = 0;
    while (lo < hi) {
        const uint64_t mid = lo + (hi - lo + 1) / 2;
        if (need(mid) <= budget) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// The pass columns: one pass's rows on the device, the job's key/value columns in d_col[0..8), `cap` rows each.  The
// split and unpack kernels write them through out(); the pipeline reads them through as_input().
struct PassColumns {
    tad_ctx *ctx;
    const tad_job *job;
    uint64_t cap = 0;
    PassColumns(tad_ctx *c, const tad_job *j) : ctx(c), job(j) {}
    PassCols out() const
    {
        const DevBuf *d = ctx->d_col;
        return PassCols{(uint32_t *)d[0].p, (uint32_t *)d[1].p, (uint32_t *)d[5].p, (uint32_t *)d[6].p,
                        (uint16_t *)d[2].p, (uint16_t *)d[3].p, (uint8_t *)d[4].p, (uint64_t *)d[7].p};
    }
    // room for `rows` rows; `carry`: the first `keep` rows are carried over (the new buffer is allocated before the old
    // one is freed), else the rows held are not kept
    void size(uint64_t rows, bool carry = false, uint64_t keep = 0)
    {
        for (int i = 0; i < 8; i++)
            if (has_col(job, i) && carry) grow_keep(ctx, ctx->d_col[i], col_bytes(i, rows), col_bytes(i, keep), ctx->stream);
            else if (has_col(job, i)) ensure(ctx, ctx->d_col[i], col_bytes(i, rows));
        cap = rows;
    }
    // the columns freed (cap 0): a split into them only counts
    void drop()
    {
        CU(cudaStreamSynchronize(ctx->stream));
        for (int i = 0; i < 8; i++) free_buf(ctx, ctx->d_col[i]);
        cap = 0;
    }
    // a column the job does not have was never allocated: its pointer is null
    tad_columns as_input(uint64_t rows) const
    {
        const PassCols o = out();
        return tad_columns{rows, rows, TAD_MEM_DEVICE, 0, o.src_ip, o.dst_ip, o.src_port, o.dst_port, o.proto,
                           o.flow_start, o.flow_end, o.value, nullptr, nullptr};
    }
};

// ---- one streamed round (run_passes, run_passes_multi) -------------------------------------------------------------------
// first() waits for the round's first block, or for its end, before the job is planned: the job's column set is that
// block's.  run() takes every block of the round: block(b, tx) enqueues the block's reads and returns the stream they end
// on; block k is released (its push returns) once block k+1 is enqueued and k's reads are done.  A rank stream job reads
// its board between blocks and ends its round early on a peer's stop (`stopper`: that rank), as next_block does on its
// own cancel; it releases every block it took before it meets its peers, so its caller's calls return at once.
struct StreamRound {
    tad_ctx *ctx;
    tad_job *job;
    tad_columns pend{};
    tad_text_column pend_txt[4]{};
    bool have_pend = false;
    int stopper = -1;

    bool first() { return have_pend = next_block(job, pend, pend_txt); }

    template <class Block>
    uint64_t run(Block block)
    {
        uint64_t rows = 0, k = 0;
        tad_columns b{};
        tad_text_column tx[4]{};
        bool got = have_pend ? (b = pend, std::copy(pend_txt, pend_txt + 4, tx), true) : next_block(job, b, tx);
        have_pend = false;
        while (got) {
            CU(cudaEventRecord(ctx->blk_ev[k & 1], block(b, (const tad_text_column *)tx)));
            if (k > 0) {
                CU(cudaEventSynchronize(ctx->blk_ev[(k - 1) & 1]));
                release_blocks(job, taken() - 1);
            }
            rows += b.rows;
            k++;
            if (job->rank_stream && stopper < 0 && (stopper = board_stop(ctx, job)) >= 0) {
                std::lock_guard<std::mutex> lk(job->mu);
                job->peer_stop.store(1);
                job->cv.notify_all();
            }
            got = next_block(job, b, tx);
        }
        if (job->rank_stream && k) {
            CU(cudaEventSynchronize(ctx->blk_ev[(k - 1) & 1]));
            release_blocks(job, taken());
        }
        return rows;
    }
    uint64_t taken()
    {
        std::lock_guard<std::mutex> lk(job->mu);
        return job->in.taken;
    }
};

// The first streamed round's pass columns: sized from the hint before it, grown geometrically up to `cap` rows while it
// arrives, the rows held carried over.  `ub` bounds the rows written so far; a block that could pass the columns has the
// cursor read back first.  `guarded` (beside the text key dictionaries; on a rank, which may not fail alone): where the
// growth does not fit the budget, the columns are dropped and the rest of the round is only counted.
struct RoundGrowth {
    tad_ctx *ctx;
    PassColumns &pc;
    const unsigned long long *d_cursor;
    uint64_t cap;
    bool to_store;                   // with a host row store: rows past `cap` go there
    bool guarded;
    bool &count_only;
    uint64_t ub = 0, have = 0;       // bound of the rows in the pass columns; the rows they hold (read back)

    // room for every row the next `n` input rows can add; false (to_store) when they would pass `cap`
    bool room(uint64_t n)
    {
        if ((pc.cap >= cap && !to_store) || ub + n <= pc.cap) { ub += n; return true; }
        CU(cudaMemcpyAsync(ctx->h_small + tad_ctx::kWPassCursor, d_cursor, 8, cudaMemcpyDeviceToHost, ctx->stream));
        CU(cudaStreamSynchronize(ctx->stream));
        have = std::min<uint64_t>(ctx->h_small[tad_ctx::kWPassCursor], pc.cap);
        if (to_store && have + n > cap) return false;
        if (have + n > pc.cap) {
            const uint64_t want = std::min(cap, std::max(2 * pc.cap, have + n));
            if (guarded) {
                size_t grow = 0;
                for (int i = 0; i < 8; i++) grow += has_col(pc.job, i) ? exact_bytes(col_bytes(i, want)) : 0;
                if (!can_grow(ctx, grow) || ctx->debug_no_grow) {
                    pc.drop();
                    count_only = true;
                    return true;
                }
            }
            pc.size(want, true, have);
        }
        ub = have + n;
        return true;
    }
};

// ---- text key slots (DESIGN.md section 10, "Text keys on the device") -------------------------------------------------
// A host chunk's text slot is copied (its marks, then the bytes of its 32-row segments) into the text staging and
// encoded into the chunk's staged u32 key column on the copy stream, ahead of the chunk's split or pack.  The
// dictionaries (ctx->tdict) live for the whole job, so ids are the same in every round.  A namespace text slot is staged
// the same way and tested against the ignore list (ctx->nsl) into the chunk's staged namespace column, in every round.
struct TextKeys {
    tad_ctx *ctx;
    tad_job *job;
    uint64_t budget;                 // the job's memory budget (messages)
    size_t tmarks;                   // the text staging's marks part: a chunk's marks; its text bytes follow
    int mark;                        // a filtered job: the slot (1 / 2) whose ids carry the drop bit; 0: none
    bool ns;                         // the ignore list filters rows: the namespace text slots are tested
    uint64_t &launches;
    bool frozen = false;             // later rounds look names up and add none
    PassColumns *yield = nullptr;    // the first round's pass columns: under the budget they give way to the dictionaries

    size_t dict_bytes() const
    {
        size_t b = 0;
        for (auto &t : ctx->tdict)
            for (DevBuf *x : t.bufs()) b += x->cap;
        return b;
    }
    // room for `extra` more dictionary bytes under the budget: in the first round the pass columns give way
    void room(size_t extra)
    {
        if (can_grow(ctx, extra)) return;
        if (yield && yield->cap) yield->drop();
        if (!can_grow(ctx, extra))
            fail(TAD_ERR_NOMEM, "the text key dictionaries need %zu bytes of device workspace (%zu held); with the job's "
                 "staging that passes the memory budget of %llu bytes", dict_bytes() + extra, dict_bytes(),
                 (unsigned long long)budget);
    }
    TextDict dict(int t) const
    {
        auto &d = ctx->tdict[t];
        return TextDict{(unsigned long long *)d.slots.p, (uint32_t *)d.minrow.p, (uint32_t *)d.slot_id.p, d.cap,
                        (uint8_t *)d.arena.p, (uint64_t *)d.off.p, (uint64_t *)d.hash.p, (unsigned long long *)d.state.p,
                        frozen ? 1u : 0u, ctx->text_mask};
    }
    // text slot t is read: a key slot, or a namespace slot of a job whose ignore list filters rows
    bool read(int t) const { return job->text[t] && (t < 2 || ns); }
    // the dictionaries' names and bytes (exact again), and the decode error flags of every slot
    void sync()
    {
        for (int t = 0; t < 2; t++)
            if (ctx->tdict[t].state.p)
                CU(cudaMemcpyAsync(ctx->h_small + tad_ctx::kWTextState + 8 * t, ctx->tdict[t].state.p, 8 * 8,
                                   cudaMemcpyDeviceToHost, ctx->copy_stream));
        const bool nst = read(2) || read(3);
        unsigned long long *w_ns = ctx->h_small + tad_ctx::kWTextState + 16;
        if (nst) CU(cudaMemcpyAsync(w_ns, ctx->nsl.p, kNsStateWords * 8, cudaMemcpyDeviceToHost, ctx->copy_stream));
        CU(cudaStreamSynchronize(ctx->copy_stream));
        for (int t = 0; t < 2 && nst; t++)
            if (w_ns[8 * t + 2])
                fail(TAD_ERR_INVALID_ARG, "invalid request: the %s text column of a streamed block does not match its marks "
                     "(a VarUInt length runs past a mark or the column's end)", t ? "dst_ns" : "src_ns");
        for (int t = 0; t < 2; t++) {
            auto &d = ctx->tdict[t];
            if (!d.state.p) continue;
            const unsigned long long *w = ctx->h_small + tad_ctx::kWTextState + 8 * t;
            if (w[2])
                fail(TAD_ERR_INVALID_ARG, "invalid request: the %s text column of a streamed block does not match its marks "
                     "(a VarUInt length runs past a mark or the column's end)", t ? "dst_ip" : "src_ip");
            if (w[5])
                fail(TAD_ERR_INVALID_ARG, "a later round of the input brought a %s name the first round did not: the "
                     "source changed between reads", t ? "dst_ip" : "src_ip");
            d.names_ub = w[0];
            d.bytes_ub = w[1];
        }
    }
    void grow_buf(DevBuf &b, size_t bytes, size_t keep)
    {
        if (bytes <= b.cap) return;
        // geometric growth where the budget allows it, else the exact size
        if (can_grow(ctx, exact_bytes(2 * b.cap))) bytes = std::max(bytes, 2 * b.cap);
        room(exact_bytes(bytes));
        grow_keep(ctx, b, bytes, keep, ctx->copy_stream);
    }
    // slot t's dictionary takes `n` more rows of `span` text bytes: its load stays at or below 1/2 counting every row as
    // a new name
    void grow(int t, uint64_t n, uint64_t span)
    {
        auto &d = ctx->tdict[t];
        auto ok = [&]() {
            const uint64_t nn = d.names_ub + n;
            return d.cap && 2 * nn <= d.cap && d.arena.cap >= d.bytes_ub + span && d.off.cap >= (nn + 1) * 8 &&
                   d.hash.cap >= nn * 8 && (!job->name_op[t] || d.keep.cap >= nn);
        };
        if (!ok()) {
            if (!d.state.p) {                     // the job's first text chunk of this slot
                d.names_ub = d.bytes_ub = 0;
                room(exact_bytes(64));
                ensure(ctx, d.state, 64);
                CU(cudaMemsetAsync(d.state.p, 0, 64, ctx->copy_stream));
                grow_buf(d.off, 4096, 0);
                CU(cudaMemsetAsync(d.off.p, 0, 8, ctx->copy_stream));
                if (const size_t m = job->name_pat[t].size()) {     // the predicate's pattern, for the match kernel
                    room(exact_bytes(m));
                    ensure(ctx, d.pat, m);
                    CU(cudaMemcpyAsync(d.pat.p, job->name_pat[t].data(), m, cudaMemcpyHostToDevice, ctx->copy_stream));
                }
            } else {
                sync();
            }
            const uint64_t names = d.names_ub, bytes = d.bytes_ub, nn = names + n;
            if (nn > (1ull << 30))
                fail(TAD_ERR_INVALID_ARG, "invalid request: a text key slot may hold at most 2^30 distinct names");
            grow_buf(d.off, (nn + 1) * 8, (names + 1) * 8);
            grow_buf(d.hash, std::max<uint64_t>(nn, 512) * 8, names * 8);
            if (job->name_op[t]) grow_buf(d.keep, std::max<uint64_t>(nn, 4096), names);
            grow_buf(d.arena, std::max<uint64_t>(bytes + span, 4096), bytes);
            if (!d.cap || 2 * nn > d.cap) {       // a larger table, the names re-inserted on the device
                uint64_t c = 1024;                // nn <= 2^30: c <= 2^31
                while (c < 2 * nn) c *= 2;
                room(exact_bytes((size_t)c * 8) + 2 * exact_bytes((size_t)c * 4));
                DevBuf ns, nm, ni;
                ensure(ctx, ns, (size_t)c * 8);
                ensure(ctx, nm, (size_t)c * 4);
                ensure(ctx, ni, (size_t)c * 4);
                TextDict old = dict(t), nd = old;
                nd.slots = (unsigned long long *)ns.p;
                nd.minrow = (uint32_t *)nm.p;
                nd.slot_id = (uint32_t *)ni.p;
                nd.cap = (uint32_t)c;
                CU(launch_text_clear(ctx->copy_stream, nd));
                CU(launch_text_rehash(ctx->copy_stream, old, nd, names));
                launches += names ? 1 : 0;
                CU(cudaStreamSynchronize(ctx->copy_stream));
                free_buf(ctx, d.slots);
                free_buf(ctx, d.minrow);
                free_buf(ctx, d.slot_id);
                d.slots = ns;
                d.minrow = nm;
                d.slot_id = ni;
                d.cap = (uint32_t)c;
            }
        }
        d.names_ub += n;
        d.bytes_ub += span;
    }
    // segment s's first byte in text slot t of a block of `rows` rows (the column's end for s = its segment count)
    static uint64_t mark_at(const tad_text_column &tx, uint64_t rows, uint64_t s)
    {
        return s < (rows + 31) / 32 ? tx.marks[s] : tx.nbytes;
    }
    // rows [lo, lo + n) of a block, cut at a mark where a slot's text does not fit the text staging; the staging grows
    // for a single segment larger than it
    uint64_t fit(const tad_text_column *tx, uint64_t rows, uint64_t lo, uint64_t n)
    {
        for (int t = 0; t < 4; t++) {
            if (!read(t)) continue;
            const uint64_t s0 = lo / 32;
            uint64_t s1 = std::min((rows + 31) / 32, (lo + n + 31) / 32);
            const uint64_t room_b = ctx->tstage.cap - tmarks, a = mark_at(tx[t], rows, s0);
            if (mark_at(tx[t], rows, s1) - a <= room_b) continue;
            const uint64_t one = mark_at(tx[t], rows, s0 + 1) - a;
            if (one > room_b) {
                CU(cudaStreamSynchronize(ctx->copy_stream));
                if (!fits(ctx, ctx->tstage, tmarks + one))
                    fail(TAD_ERR_NOMEM, "32 rows of a text column hold %llu bytes: more than the memory budget of %llu "
                         "bytes leaves for the text staging", (unsigned long long)one, (unsigned long long)budget);
                ensure(ctx, ctx->tstage, tmarks + one);
                s1 = s0 + 1;
            } else {
                uint64_t l = s0 + 1, h = s1;
                while (l < h) {
                    const uint64_t mid = l + (h - l + 1) / 2;
                    if (mark_at(tx[t], rows, mid) - a <= room_b) l = mid; else h = mid - 1;
                }
                s1 = l;
            }
            n = std::min(n, s1 * 32 - lo);
        }
        return n;
    }
    // text slots of rows [lo, lo + n) of a block of `rows` rows -> their ids in the chunk's staged key columns `c`, and
    // the ignore list's verdicts in its staged namespace columns.  A filtered job then marks the rows its predicates drop
    // (the first round also evaluates them on the names the chunk added) using the chunk's staged proto column.
    void encode(const tad_text_column *tx, uint64_t rows, uint64_t lo, uint64_t n, const ColPtrs &c)
    {
        uint32_t *dst[4] = {job->text[0] ? const_cast<uint32_t *>(c.src_ip) : nullptr,
                            job->text[1] ? const_cast<uint32_t *>(c.dst_ip) : nullptr,
                            const_cast<uint32_t *>(c.src_ns), const_cast<uint32_t *>(c.dst_ns)};
        for (int t = 0; t < 4; t++) {
            if (!read(t)) continue;
            const uint64_t s0 = lo / 32, s1 = std::min((rows + 31) / 32, (lo + n + 31) / 32);
            const uint64_t a = mark_at(tx[t], rows, s0), span = mark_at(tx[t], rows, s1) - a;
            // the first round builds the dictionary; later rounds look names up in it and add none (a frozen table
            // needs no room: a missing name fails the round)
            if (t < 2 && (!frozen || !ctx->tdict[t].state.p)) grow(t, n, span);
            char *m = static_cast<char *>(ctx->tstage.p);
            CU(cudaMemcpyAsync(m, tx[t].marks + s0, (s1 - s0) * 8, cudaMemcpyHostToDevice, ctx->copy_stream));
            if (span) CU(cudaMemcpyAsync(m + tmarks, tx[t].bytes + a, span, cudaMemcpyHostToDevice, ctx->copy_stream));
            if (t >= 2) {                         // a namespace: no dictionary, the row's verdict only
                CU(launch_ns_match(ctx->copy_stream, ctx->nsl.p, job->ns_names, job->ns_image.size(), ctx->text_mask,
                                   static_cast<unsigned long long *>(ctx->nsl.p) + 8 * (t - 2),
                                   reinterpret_cast<const uint8_t *>(m + tmarks), span, reinterpret_cast<const uint64_t *>(m),
                                   (uint32_t)(s1 - s0), s0 * 32, rows, lo, n, ctx->tscratch.p, ctx->tscratch.cap, dst[t]));
                launches += kNsLaunches;
                continue;
            }
            CU(launch_text_encode(ctx->copy_stream, dict(t), reinterpret_cast<const uint8_t *>(m + tmarks), span,
                                  reinterpret_cast<const uint64_t *>(m), (uint32_t)(s1 - s0), s0 * 32, rows, lo, n,
                                  ctx->tscratch.p, ctx->tscratch.cap, dst[t]));
            launches += kTextLaunches;
            if (job->name_op[t] && !frozen) {     // an open dictionary: its new names get their predicate byte
                auto &d = ctx->tdict[t];
                CU(launch_text_match(ctx->copy_stream, dict(t), (uint8_t *)d.keep.p, job->name_op[t],
                                     (const uint8_t *)d.pat.p, (uint32_t)job->name_pat[t].size(), n));
                launches++;
            }
        }
        if (mark) {
            TextMark m{};
            for (int t = 0; t < 2; t++) {
                m.ids[t] = dst[t];
                m.keep[t] = job->name_op[t] ? (const uint8_t *)ctx->tdict[t].keep.p : nullptr;
            }
            m.proto = c.proto;
            m.proto_eq = job->proto_eq;
            m.mark = dst[mark - 1];
            CU(launch_text_mark(ctx->copy_stream, m, n));
            launches++;
        }
    }
    // each text slot's dictionary to host memory the job owns (tad_job_names); the device copy goes with the workspace
    void export_names()
    {
        sync();
        for (int t = 0; t < 2; t++) {
            if (!job->text[t]) continue;
            auto &d = ctx->tdict[t];
            const uint64_t names = d.state.p ? d.names_ub : 0, bytes = d.state.p ? d.bytes_ub : 0;
            job->names[t].resize(bytes);
            job->names_off[t].assign(names + 1, 0);
            if (bytes) CU(cudaMemcpy(job->names[t].data(), d.arena.p, bytes, cudaMemcpyDeviceToHost));
            if (names) CU(cudaMemcpy(job->names_off[t].data(), d.off.p, (names + 1) * 8, cudaMemcpyDeviceToHost));
        }
        CU(release(ctx));
    }
    // A dictionary lives for one job.  Every buffer is freed, also on a context with a sticky error (a failed job's
    // cleanup); returns the first error.
    static cudaError_t release(tad_ctx *ctx) { return free_bufs(ctx, kJobs); }
};

// One sweep over a job's input for pass (v, M): the rows that pass the job's filters are counted per residue (per owner
// rank and residue on several GPUs) and the pass's rows are split into the pass columns.  Host blocks go through two
// staging halves of `chunk` rows each, the split of every chunk behind its copy on the copy stream.
struct Sweep {
    tad_ctx *ctx;
    const tad_job *job;
    PassOut &acc;
    const bool ns;                   // the ns_ignore list filters rows: the namespace columns are staged too
    uint64_t chunk = 0;              // rows per staging half; 0: no host input
    size_t half_bytes = 0;
    RowFilter f{};
    unsigned long long *cnt = nullptr, *cursor = nullptr;   // the split's counters and the pass columns' cursor
    int log_world = 0;               // as launch_pass_split takes it
    const int mark;                  // a filtered job: the slot (1 / 2) whose ids carry the drop bit (host chunks only)
    TextKeys *text = nullptr;        // the job's text key slots, encoded into the staged key columns
    uint64_t nchunk = 0;             // host chunks staged in this sweep
    bool any_host = false;
    double lent0 = 0;                // the job's lent time when the sweep began (lend)

    // `text_row`: text staging and encode scratch bytes per staged row, planned into the staging's 1/16 of the budget
    Sweep(tad_ctx *c, const tad_job *j, PassOut &a, bool host_input, uint64_t budget, size_t text_row)
        : ctx(c), job(j), acc(a), ns(!j->ns_ignore.empty() && (has_col(j, 8) || has_col(j, 9))),
          mark(j->filtered() ? (j->text[0] ? 1 : 2) : 0)
    {
        size_t row_bytes = 0;
        for (int i = 0; i < 10; i++) row_bytes += staged(i) ? col_bytes(i, 1) : 0;
        if (host_input && row_bytes) {
            chunk = std::min<uint64_t>(8u << 20, std::max<uint64_t>(2048, budget / 16 / (2 * row_bytes + text_row))) &
                    ~uint64_t(2047);
            for (int i = 0; i < 10; i++) half_bytes += staged(i) ? exact_bytes(col_bytes(i, chunk)) : 0;
        }
    }
    bool staged(int i) const { return has_col(job, i) && (i < 8 || ns); }
    size_t stage_bytes() const { return 2 * half_bytes; }

    // staging half h from row `at` as kernel input, with rows [lo, lo + n) of block `b` copied there on the copy stream
    // (a null `b`: none); text slots are left to the encoder (TextKeys)
    ColPtrs stage(const tad_columns *b, uint64_t lo, uint64_t n, int h, uint64_t at) const
    {
        ColPtrs c{};
        char *dst = static_cast<char *>(ctx->stage.p) + h * half_bytes;
        for (int i = 0; i < 10; i++) {
            if (!staged(i)) continue;
            char *d = dst + col_bytes(i, at);
            if (b && !is_text(job, i))
                CU(cudaMemcpyAsync(d, static_cast<const char *>(col_ptr(*b, i)) + col_bytes(i, lo), col_bytes(i, n),
                                   b->mem == TAD_MEM_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice,
                                   ctx->copy_stream));
            set_col(c, i, d);
            dst += exact_bytes(col_bytes(i, chunk));
        }
        return c;
    }
    // the sweep's start (its counters are reset by the caller): the pass columns' previous readers are done before the
    // copy stream writes again
    void begin(bool host_input)
    {
        CU(cudaEventRecord(ctx->ev[0], ctx->stream));
        nchunk = 0;
        any_host = false;
        lent0 = job->lent_ms;
        if (host_input) {
            CU(cudaEventRecord(ctx->start_ev, ctx->stream));
            CU(cudaStreamWaitEvent(ctx->copy_stream, ctx->start_ev, 0));
        }
    }
    // enqueue the split of rows [from, b.rows) of block `b` (a table, or one block of a streamed round; text slots: `tx`)
    // for pass (v, M) into `pc`; `count_only`: the rows are only counted
    void feed(const tad_columns &b, uint64_t from, uint32_t v, uint32_t M, const PassColumns &pc, bool count_only,
              const tad_text_column *tx)
    {
        cudaStream_t st = ctx->stream;
        if (from >= b.rows) return;
        if (b.mem == TAD_MEM_DEVICE) {
            CU(launch_pass_split(st, offset_cols(col_ptrs(b), from), b.rows - from, f, M - 1, v, pc.out(),
                                 count_only ? 0u : (uint32_t)pc.cap, cursor, cnt, 0, log_world));
            acc.launches++;
            return;
        }
        any_host = true;
        ensure(ctx, ctx->stage, stage_bytes());
        for (uint64_t lo = from, n; lo < b.rows; lo += n, nchunk++) {
            n = std::min<uint64_t>(chunk, b.rows - lo);
            if (text) n = text->fit(tx, b.rows, lo, n);
            const int h = (int)(nchunk & 1);
            if (nchunk >= 2) CU(cudaStreamWaitEvent(ctx->copy_stream, ctx->stage_ev[h], 0));   // split of chunk k-2 is done
            const ColPtrs c = stage(&b, lo, n, h, 0);
            if (text) text->encode(tx, b.rows, lo, n, c);
            CU(cudaEventRecord(ctx->chunk_ev[h], ctx->copy_stream));
            CU(cudaStreamWaitEvent(st, ctx->chunk_ev[h], 0));
            CU(launch_pass_split(st, c, n, f, M - 1, v, pc.out(), count_only ? 0u : (uint32_t)pc.cap, cursor, cnt, mark,
                                 log_world));
            acc.launches++;
            CU(cudaEventRecord(ctx->stage_ev[h], st));
        }
    }
    // the sweep's end: its time goes to the h2d phase where it staged host rows (the split runs behind the copies), the
    // time the job lent the GPU meanwhile left out; `counts`: the counters and the cursor are copied to h_small
    void end(bool counts)
    {
        CU(cudaEventRecord(ctx->ev[1], ctx->stream));
        if (counts) CU(cudaMemcpyAsync(ctx->h_small, cnt, (kMaxPasses + 1) * 8, cudaMemcpyDeviceToHost, ctx->stream));
        CU(cudaStreamSynchronize(ctx->stream));
        float ms = 0;
        CU(cudaEventElapsedTime(&ms, ctx->ev[0], ctx->ev[1]));
        ms = (float)std::max(0.0, ms - (job->lent_ms - lent0));
        acc.phase_ms[any_host ? TAD_PHASE_H2D : TAD_PHASE_SCATTER] += ms;
        acc.device_ms += ms;
    }
};

// ---- host row store (DESIGN.md section 11) ----------------------------------------------------------------------------
// One job's rows in the store: per low-hash-bit residue, a list of pages filled in order.  The pages go back to the
// context when the job ends, however it ends.  The first round's blocks are packed into the staging halves; every full
// half (and the last, partial one) is counted, scanned and scattered per residue into an out-stage half, whose residue
// segments are then copied to the residue's pages on the D2H stream.  The passes load their residues from the pages.
struct RowStore {
    tad_ctx *ctx;
    std::vector<char *> pages[kMaxPasses];
    uint64_t rows[kMaxPasses] = {};
    bool active = false;             // the current round goes to the store
    Sweep *sw;                       // the round's staging, filter and counters
    uint64_t budget;                 // the job's host budget
    size_t scratch_bytes;
    uint64_t fill = 0, nhalf = 0, npack = 0;   // rows in the staging half being filled; halves filled; out-stage halves used
    int opend = -1;                  // out-stage half whose copies to the store are not issued yet
    Row32 *ost[2] = {nullptr, nullptr};
    void *pscratch = nullptr;
    uint32_t *d_chunk = nullptr;
    RowStore(tad_ctx *c, Sweep &s, uint64_t host_budget, size_t pack_scratch)
        : ctx(c), sw(&s), budget(host_budget), scratch_bytes(pack_scratch) {}
    void clear()
    {
        cudaStreamSynchronize(ctx->d2h_stream);       // no copy into a page is still in flight
        for (int j = 0; j < kMaxPasses; j++) {
            ctx->store_free.insert(ctx->store_free.end(), pages[j].begin(), pages[j].end());
            pages[j].clear();
            rows[j] = 0;
        }
    }
    ~RowStore() { clear(); }
    // the out-stage: two halves of `chunk` packed rows, the pack scratch and the chunk counts
    void start(size_t ostage_bytes)
    {
        ensure(ctx, ctx->stage, sw->stage_bytes());
        ensure(ctx, ctx->ostage, ostage_bytes);
        char *p = static_cast<char *>(ctx->ostage.p);
        ost[0] = reinterpret_cast<Row32 *>(p);
        ost[1] = reinterpret_cast<Row32 *>(p + sw->chunk * sizeof(Row32));
        pscratch = p + 2 * sw->chunk * sizeof(Row32);
        d_chunk = reinterpret_cast<uint32_t *>(p + 2 * sw->chunk * sizeof(Row32) + scratch_bytes);
        active = true;
    }
    // fallback: the pages go back to the context
    void drop()
    {
        CU(cudaStreamSynchronize(ctx->stream));      // no pack reads the staging halves any more
        clear();
        active = false;
        opend = -1;
    }
    // copies of out-stage half `o`'s residue segments to the pages; false when the store would pass its budget
    bool out(int o)
    {
        const uint64_t page_rows = ctx->store_page / sizeof(Row32);
        CU(cudaEventSynchronize(ctx->cnt_ev[o]));
        CU(cudaStreamWaitEvent(ctx->d2h_stream, ctx->cnt_ev[o], 0));
        const uint32_t *n = ctx->h_chunk + kMaxPasses * o;
        uint64_t at = 0;
        for (int j = 0; j < kMaxPasses; j++) {
            for (uint64_t left = n[j]; left;) {
                const uint64_t used = rows[j] % page_rows;
                if (used == 0) {
                    char *p = store_take_page(ctx, budget);
                    if (!p) return false;
                    pages[j].push_back(p);
                }
                const uint64_t k = std::min(left, page_rows - used);
                CU(cudaMemcpyAsync(pages[j].back() + used * sizeof(Row32), ost[o] + at, k * sizeof(Row32),
                                   cudaMemcpyDeviceToHost, ctx->d2h_stream));
                rows[j] += k;
                at += k;
                left -= k;
            }
        }
        CU(cudaEventRecord(ctx->ost_ev[o], ctx->d2h_stream));
        return true;
    }
    // count / scan / scatter `n` <= chunk device rows into the next out-stage half, then issue the copies of the previous
    // one (its counts are back by now; this chunk's copies are on the bus meanwhile).  `totals`: count them for the job.
    // `totals` also tells staged rows (marked rows of a filtered job among them) from the pass columns' clean ones.
    void pack(const ColPtrs &c, uint64_t n, bool totals)
    {
        const int o = (int)(npack++ & 1);
        cudaStream_t st = ctx->stream;
        CU(cudaStreamWaitEvent(st, ctx->ost_ev[o], 0));      // the copies that last read out-stage half o are done
        CU(launch_residue_pack(st, c, n, sw->f, pscratch, scratch_bytes, d_chunk, totals ? sw->cnt : nullptr, ost[o],
                               totals ? sw->mark : 0));
        sw->acc.launches += 3;
        CU(cudaMemcpyAsync(ctx->h_chunk + kMaxPasses * o, d_chunk, kMaxPasses * 4, cudaMemcpyDeviceToHost, st));
        CU(cudaEventRecord(ctx->cnt_ev[o], st));
        if (opend >= 0 && !out(opend)) { drop(); return; }
        opend = o;
    }
    void pack_half()                 // the staging half being filled
    {
        const int h = (int)(nhalf++ & 1);
        CU(cudaEventRecord(ctx->chunk_ev[h], ctx->copy_stream));
        CU(cudaStreamWaitEvent(ctx->stream, ctx->chunk_ev[h], 0));
        pack(sw->stage(nullptr, 0, 0, h, 0), fill, true);
        CU(cudaEventRecord(ctx->stage_ev[h], ctx->stream));
        fill = 0;
    }
    // one block into the staging halves (a D2D copy for a device block); a full half is packed.  Returns the rows it
    // took: the store may fall back inside the block.
    uint64_t put(const tad_columns &b, const tad_text_column *tx)
    {
        uint64_t lo = 0;
        sw->any_host = true;         // the round's time is the copies' (h2d phase), as for a sweep of host blocks
        while (lo < b.rows && active) {
            if (sw->job->cancel.load()) fail(TAD_ERR_CANCELLED, "job cancelled");
            const int h = (int)(nhalf & 1);
            if (fill == 0) CU(cudaStreamWaitEvent(ctx->copy_stream, ctx->stage_ev[h], 0));   // its last pack is done
            uint64_t n = std::min(sw->chunk - fill, b.rows - lo);
            if (sw->text) n = sw->text->fit(tx, b.rows, lo, n);
            const ColPtrs c = sw->stage(&b, lo, n, h, fill);
            if (sw->text) sw->text->encode(tx, b.rows, lo, n, c);
            fill += n;
            lo += n;
            if (fill == sw->chunk) pack_half();
        }
        return lo;
    }
    // end of the round: the last half, the last copies; the out-stage is not needed any more.  True when the store
    // holds the whole round.
    bool end()
    {
        if (active && fill) pack_half();
        if (active && opend >= 0 && !out(opend)) drop();
        const bool stored = active;
        if (active && opend >= 0) CU(cudaStreamWaitEvent(ctx->stream, ctx->ost_ev[opend], 0));
        active = false;
        CU(cudaStreamSynchronize(ctx->stream));
        free_buf(ctx, ctx->ostage);
        return stored;
    }
    // pass (v, M) from the store into the pass columns, through the staging halves
    void load(uint32_t v, uint32_t M, const PassCols &to)
    {
        const uint64_t page_rows = ctx->store_page / sizeof(Row32), piece = sw->half_bytes / sizeof(Row32);
        sw->begin(true);
        sw->any_host = true;
        uint64_t at = 0, k = 0;
        for (uint32_t j = v; j < (uint32_t)kMaxPasses; j += M)
            for (size_t pg = 0; pg < pages[j].size(); pg++) {
                const uint64_t in_pg = std::min(page_rows, rows[j] - pg * page_rows);
                for (uint64_t r0 = 0; r0 < in_pg; r0 += piece, k++) {
                    const uint64_t n = std::min(piece, in_pg - r0);
                    const int h = (int)(k & 1);
                    Row32 *dst = reinterpret_cast<Row32 *>(static_cast<char *>(ctx->stage.p) + h * sw->half_bytes);
                    CU(cudaStreamWaitEvent(ctx->copy_stream, ctx->stage_ev[h], 0));    // its last unpack is done
                    CU(cudaMemcpyAsync(dst, pages[j][pg] + r0 * sizeof(Row32), n * sizeof(Row32),
                                       cudaMemcpyHostToDevice, ctx->copy_stream));
                    CU(cudaEventRecord(ctx->chunk_ev[h], ctx->copy_stream));
                    CU(cudaStreamWaitEvent(ctx->stream, ctx->chunk_ev[h], 0));
                    CU(launch_store_unpack(ctx->stream, dst, n, to, at));
                    sw->acc.launches++;
                    CU(cudaEventRecord(ctx->stage_ev[h], ctx->stream));
                    at += n;
                }
            }
        sw->end(false);
    }
};

// The buffers earlier passes grew are freed, except what every pass reads (kPasses).
void free_pass_buffers(tad_ctx *ctx) { CU(free_bufs(ctx, kPasses)); }

using PassList = std::deque<std::pair<uint32_t, uint32_t>>;

// The passes of a job in hash-range passes: (v, P) for v < P, in order, each run by run(v, M, rest, out) with `rest` the
// passes queued behind it; an empty pass leaves `out` as it is.  A pass for which run returns true (split) is replaced by
// (v, 2M) and (v + M, 2M) and gives its fits back.  Fills `acc` (sums over the passes, acc.block = all result rows) and
// returns the number of passes.
template <class Run>
uint32_t run_pass_queue(tad_ctx *ctx, tad_job *job, uint32_t P, PassOut &acc, Run run)
{
    PassList todo;
    for (uint32_t v = 0; v < P; v++) todo.push_back({v, P});
    std::vector<PassOut> outs;
    uint32_t passes = 0, planned = P;
    set_passes(job, 0, planned);
    try {
        while (!todo.empty()) {
            const tad_progress before = progress_of(job);
            const uint32_t v = todo.front().first, M = todo.front().second;
            todo.pop_front();
            PassOut o;
            if (run(v, M, (const PassList &)todo, o)) {
                todo.push_front({v + M, 2 * M});
                todo.push_front({v, 2 * M});
                set_passes(job, passes, ++planned, &before);
                continue;
            }
            add_pass(acc, o);
            if (o.block.p) outs.push_back(o);
            set_passes(job, ++passes, planned);
        }
        join_passes(ctx, outs, acc);
    } catch (...) {
        for (PassOut &o : outs) give_pinned(ctx, o.block);
        throw;
    }
    return passes;
}

// A single-GPU job in hash-range passes (DESIGN.md sections 9 and 10).  Pass (v, M) holds the rows whose key hash has
// (h & (M - 1)) == v.  The first sweep counts the rows of every residue mod 64, which sizes every pass of every M exactly;
// a pass whose spill scratch or result buffer turns out not to fit is split into (v, 2M) and (v + M, 2M).  A sweep reads
// the job's columns (device-resident: one split launch; host: double-buffered chunks behind the copies) or, for a
// streamed job, the blocks of one round.  Every later sweep must count what the first one counted.
// Fills `acc` (sums over passes, acc.block = all result rows) and returns the number of passes.  `shared`: a job run while
// an ARIMA pass is parked (interleave), whose last round stays open until its passes are done.
uint32_t run_passes(tad_ctx *ctx, tad_job *job, uint64_t budget, uint64_t host_budget_set, bool shared, PassOut &acc)
{
    cudaStream_t st = ctx->stream;
    const bool stream = job->stream;
    // a streamed job's column set is that of its first block: wait for it (or for an empty round) before planning
    StreamRound round{ctx, job};
    if (stream) round.first();
    const tad_columns &hc = job->cols;
    const uint64_t R = stream ? job->rows_hint : hc.rows;        // rows to plan for (0: unknown)
    const bool host_input = stream || hc.mem != TAD_MEM_DEVICE;  // a streamed round may bring host blocks
    // host input: double-buffered chunk staging, at most 1/16 of the budget; text slots: per staged row, kTextRowBytes
    // of text staging (any IPv6 text) and the encode scratch.  `text`: key slots with dictionaries; `staged_text`: those
    // or namespace text slots that an ignore list tests (no dictionary), which share the staging one slot at a time
    const bool text = job->text[0] || job->text[1];
    const bool ns_text = !job->ns_ignore.empty() && (job->text[2] || job->text[3]);
    const bool staged_text = text || ns_text;
    constexpr size_t kTextRowBytes = 48;
    Sweep sw(ctx, job, acc, host_input, budget,
             staged_text ? kTextRowBytes + text_scratch_bytes(1u << 20) / (1u << 20) + 1 : 0);
    const uint64_t chunk = sw.chunk;
    size_t tmarks = 0, text_bytes = 0;
    if (staged_text && chunk) {
        tmarks = exact_bytes((chunk / 32 + 2) * 8);
        text_bytes = alloc_bytes(tmarks + chunk * kTextRowBytes) + alloc_bytes(text_scratch_bytes(chunk));
    }
    const size_t stage_bytes = sw.stage_bytes();
    const size_t plan_stage = stage_bytes + text_bytes;      // the text staging is planned as part of the staging
    // rows one pass may hold: the largest count whose workspace (exact partition, empty workspace) fits `b`
    auto pass_cap = [&](uint64_t b) {
        return largest_fit(stream ? kMaxPassRows : std::min(R, kMaxPassRows), b,
                           [&](uint64_t n) { return pass_need(ctx, job, n, n, false, plan_stage, true); });
    };
    uint64_t cap = pass_cap(budget);
    // host row store (streamed input with a host budget, read once per job by store_trim): out-stage of two halves of
    // `chunk` packed rows.  The plan above does not depend on it; the store is used only where the out-stage fits next
    // to the round's buffers at `cap`.
    const size_t pack_scratch = stream && chunk && host_budget_set ? exact_bytes(residue_pack_scratch_bytes(chunk)) : 0;
    const size_t ostage_bytes = pack_scratch ? 2 * chunk * sizeof(Row32) + pack_scratch + 256 : 0;
    const uint64_t host_budget =
        ostage_bytes && store_round_need(ctx, job, cap, plan_stage, ostage_bytes) <= budget ? host_budget_set : 0;
    if (host_budget && ctx->store_page == 0) fail(TAD_ERR_INTERNAL, "host row store without a page size");
    if (cap == 0) fail(TAD_ERR_NOMEM, "a memory budget of %llu bytes does not hold one row of a pass", (unsigned long long)budget);
    uint32_t P = 1;
    while (P < (uint32_t)kMaxPasses && R / P > cap / 8 * 7) P *= 2;     // 1/8 head-room for hash imbalance
    // pass columns: a table's passes get `cap` rows; a streamed round's from the hint (or 1M rows without one), grown
    // geometrically up to `cap` while the first round arrives
    free_workspace(ctx);
    PassColumns pc(ctx, job);
    pc.size(stream ? std::min(cap, R ? R / P + R / P / 8 + 2048 : uint64_t(1) << 20) : cap);
    if (stage_bytes && !stream) ensure(ctx, ctx->stage, stage_bytes);
    if (text_bytes) {
        ensure(ctx, ctx->tstage, tmarks + chunk * kTextRowBytes);
        ensure(ctx, ctx->tscratch, text_scratch_bytes(chunk));
    }
    ensure(ctx, ctx->pcnt, (kMaxPasses + 1) * 8);
    ensure(ctx, ctx->stats, 64 * sizeof(uint32_t));
    unsigned long long *d_cnt = static_cast<unsigned long long *>(ctx->pcnt.p);   // [0, 64): rows per residue, [64]: pass cursor
    const unsigned long long *h_cnt = ctx->h_small;
    sw.f = row_filter(ctx, job, sw.ns);
    if (ns_text) {                   // the ignore list's names, with its decode error flags cleared
        ensure(ctx, ctx->nsl, job->ns_image.size());
        CU(cudaMemcpyAsync(ctx->nsl.p, job->ns_image.data(), job->ns_image.size(), cudaMemcpyHostToDevice, ctx->copy_stream));
    }
    sw.cnt = d_cnt;
    sw.cursor = d_cnt + kMaxPasses;
    TextKeys tk{ctx, job, budget, tmarks, sw.mark, ns_text, acc.launches, false, &pc};
    if (staged_text) sw.text = &tk;
    bool count_only = false;         // the first round's rows are only counted (the store fell back, or the pass columns
                                     // gave way to the text key dictionaries)
    uint32_t sweeps = 0;
    // first streamed round: the pass columns grow as it arrives; beside the dictionaries they may not grow past the
    // budget, and the round then only counts.  With a host budget, rows that would pass `cap` go to the host row store.
    RoundGrowth grow{ctx, pc, d_cnt + kMaxPasses, cap, host_budget != 0, text, count_only};
    RowStore rs(ctx, sw, host_budget, pack_scratch);
    bool stored = false;             // the store holds the whole first round: the passes load from it
    bool dropped = false;            // the store fell back in the first round: it only counted
    // the pass columns overflow in the first round: their `have` rows go to the store first (counted already)
    auto switch_to_store = [&]() {
        // the out-stage was planned without the dictionaries: where it does not fit beside them, the round only counts
        if (text && !can_grow(ctx, exact_bytes(ostage_bytes) + (stage_bytes > ctx->stage.cap ? exact_bytes(stage_bytes) : 0))) {
            count_only = true;
            return;
        }
        rs.start(ostage_bytes);
        const uint64_t have = grow.have;
        const ColPtrs held = col_ptrs(pc.as_input(have));
        for (uint64_t lo = 0; lo < have && rs.active; lo += chunk) rs.pack(offset_cols(held, lo), std::min(chunk, have - lo), false);
        if (!rs.active) count_only = true;   // the store fell back: the rest of the round is only counted
    };
    uint64_t counts[kMaxPasses];
    bool open = false;               // a streamed round is swept and its caller waits in tad_stream_end
    // one sweep over the input: the rows of pass (v, M) -> the pass columns; returns the rows of the pass
    auto sweep = [&](uint32_t v, uint32_t M) -> uint64_t {
        CU(cudaMemsetAsync(d_cnt, 0, (kMaxPasses + 1) * 8, st));
        sw.begin(host_input);
        if (!stream) {
            sw.feed(hc, 0, v, M, pc, count_only, nullptr);
        } else {
            grow.ub = 0;
            if (sweeps == 0 && host_budget && P > 1)         // the hint plans passes: the round goes to the store
                rs.start(ostage_bytes);
            const uint64_t rows = round.run([&](const tad_columns &b, const tad_text_column *tx) {
                // TextKeys::room drops the first round's pass columns (cap 0) for the dictionaries: the rest is only counted
                if (sweeps == 0 && pc.cap == 0 && !rs.active) count_only = true;
                if (sweeps == 0 && host_budget && !rs.active && !count_only && !grow.room(b.rows)) switch_to_store();
                else if (sweeps == 0 && !host_budget && !count_only) grow.room(b.rows);
                const bool to_store = rs.active;
                const uint64_t took = to_store ? rs.put(b, tx) : 0;
                count_only = count_only || (to_store && !rs.active);   // the store fell back: the rest is only counted
                if (!rs.active) sw.feed(b, took, v, M, pc, count_only, tx);      // (v, M) = (0, P) while it stores
                if (to_store && !rs.active) {
                    CU(cudaEventRecord(ctx->start_ev, st));
                    CU(cudaStreamWaitEvent(ctx->copy_stream, ctx->start_ev, 0));
                }
                return b.mem == TAD_MEM_DEVICE && !to_store ? st : ctx->copy_stream;
            });
            if (sweeps == 0) job->round_rows = rows;
            if (sweeps == 0 && ctx->ostage.p) {
                stored = rs.end();
                dropped = !stored;
                count_only = false;          // later rounds split their pass into the pass columns
            }
            open = true;
        }
        sw.end(true);
        if (staged_text) tk.sync();
        if (sweeps > 0)
            for (int j = 0; j < kMaxPasses; j++)
                if (h_cnt[j] != counts[j])
                    fail(TAD_ERR_INVALID_ARG, "sweep %u of the input delivered %llu filtered rows of hash residue %d, the first "
                         "delivered %llu: the source changed between reads", sweeps + 1, (unsigned long long)h_cnt[j], j,
                         (unsigned long long)counts[j]);
        sweeps++;
        tk.frozen = true;
        tk.yield = nullptr;
        return h_cnt[kMaxPasses];
    };
    const uint64_t got0 = sweep(0, P);
    for (int j = 0; j < kMaxPasses; j++) counts[j] = h_cnt[j];
    if (text) {
        count_only = false;
        // the passes run beside the dictionaries
        const size_t held_dict = tk.dict_bytes();
        cap = pass_cap(budget > held_dict ? budget - held_dict : 0);
        if (cap == 0)
            fail(TAD_ERR_NOMEM, "the text key dictionaries hold %zu bytes: beside them the memory budget of %llu bytes does "
                 "not hold one row of a pass", held_dict, (unsigned long long)budget);
    }
    auto pass_rows = [&](uint32_t v, uint32_t M) {
        uint64_t n = 0;
        for (uint32_t j = v; j < (uint32_t)kMaxPasses; j += M) n += counts[j];
        return n;
    };
    auto largest = [&](uint32_t M) {
        uint64_t m = 0;
        for (uint32_t v = 0; v < M; v++) m = std::max(m, pass_rows(v, M));
        return m;
    };
    const uint32_t P0 = P;
    if (stream) {
        // an overestimated hint must not cost a round per surplus pass: plan from the rows the first round delivered,
        // as an exact hint would have, at the price of that one round (loaded is then false unless P comes back to P0)
        uint32_t Pr = 1;
        while (Pr < (uint32_t)kMaxPasses && job->round_rows / Pr > cap / 8 * 7) Pr *= 2;
        P = stored ? Pr : std::min(P, Pr);      // stored: no round to save, so a low hint does not keep P either
    }
    while (P < (uint32_t)kMaxPasses && largest(P) > cap) P *= 2;
    auto too_big = [&](uint64_t rows) {
        fail(TAD_ERR_NOMEM, "one 1/%d hash range of the table (%llu rows) needs %zu bytes of device workspace; the memory "
             "budget is %llu bytes", kMaxPasses, (unsigned long long)rows,
             pass_need(ctx, job, rows, rows, false, plan_stage, true), (unsigned long long)budget);
    };
    if (largest(P) > cap) too_big(largest(kMaxPasses));
    bool loaded = !stored && !dropped && P == P0 && got0 <= pc.cap;     // pass (0, P) is in the pass columns already
    // a streamed round stays open until the engine knows whether another sweep (round) follows: one does while a queued
    // pass has rows that are not in the store.  A shared job's last round stays open until `done`: should a pass not fit
    // the reserve, the caller has not been told its input is complete and delivers the rows again in the job's turn.
    auto finish_round = [&](bool more, bool done = false) {
        const bool again = !stored && more;
        if (!open || (shared && !again && !done)) return;
        close_round(job, again);
        open = false;
    };
    if (stored)
        for (int j = 0; j < kMaxPasses; j++) job->stored_rows += rs.rows[j];
    if (!loaded) finish_round(largest(P) > 0);
    auto run_one = [&](uint32_t v, uint32_t M, const PassList &rest, PassOut &o) {
        const uint64_t rows = pass_rows(v, M);
        bool more = rows > 0;        // the round the previous pass was swept in closes once that pass has run
        for (const auto &e : rest) more = more || pass_rows(e.first, e.second) > 0;
        if (!loaded) finish_round(more);
        if (job->cancel.load()) fail(TAD_ERR_CANCELLED, "job cancelled");
        if (!loaded && rows) {
            if (stream && rows > pc.cap) pc.size(rows);     // later rounds: the counts size the pass columns exactly
            if (stored) rs.load(v, M, pc.out()); else sweep(v, M);
        }
        loaded = false;
        if (!rows) return false;
        // optimistic partition where its slot buffer fits next to what the context holds; else the exact one, on a
        // workspace cleared of earlier passes' buffers if need be (the planner sized `cap` for that)
        const bool opt = pass_need(ctx, job, rows, cap, true, stage_bytes, false) <= budget;
        if (!opt && pass_need(ctx, job, rows, cap, false, stage_bytes, false) > budget) free_pass_buffers(ctx);
        try {
            run_pipeline(ctx, job, pc.as_input(rows), false, !opt, o);
        } catch (const PassSplit &e) {
            CU(cudaStreamSynchronize(st));
            // the planned workspace fitted; what outgrew the budget is known only now (a result rerun, a spill)
            if (M >= (uint32_t)kMaxPasses)
                fail(TAD_ERR_NOMEM, "the %s of a 1/%d hash range of the table (%llu rows) needs %zu bytes beside the %zu bytes "
                     "of workspace the pass holds: more than the memory budget of %llu bytes", e.what, kMaxPasses,
                     (unsigned long long)rows, e.bytes, e.held, (unsigned long long)budget);
            return true;
        }
        return false;
    };
    const uint32_t passes = run_pass_queue(ctx, job, P, acc, run_one);
    finish_round(false, true);
    if (text) tk.export_names();
    return passes;
}

// ---- several GPUs in hash-range passes (DESIGN.md section 9, "Several GPUs") ---------------------------------------------
// The pipeline buffers one multi-GPU pass grows (the exported buffer apart), with upper bounds as pass_need: `rows` input
// rows of this rank, `owned` rows it owns, `global` rows over all ranks; both partitions when `slots` (an overflow falls
// back to the exact one).
std::vector<std::pair<DevBuf *, size_t>> mp_pipe_bufs(tad_ctx *ctx, const tad_job *job, uint64_t global, uint64_t rows,
                                                       uint64_t owned, bool slots)
{
    const size_t W = ctx->cfg.world_size;
    PipeShape s;
    s.rows = rows;
    s.algo = job->spec.algo;
    s.B = buckets(ctx, global);
    s.Bl = s.B >> log_world(ctx);
    s.owned = s.series = owned;
    s.out_cap = out_cap_guess(owned, (job->spec.flags & TAD_FLAG_EMIT_ALL) != 0);
    PipeSizes z = pipe_sizes(s);
    const bool pull = ctx->peer_pull && ctx->exact_pull;
    const size_t Bl = s.Bl;
    z.part = pull ? 0 : std::max<uint64_t>(rows, 1) * sizeof(Row32);
    z.entries = std::max<uint64_t>(owned, 1) * sizeof(SeriesEntry);
    z.hist = z.cursor = z.offsets = 0;      // in exact_bufs, with the most chunks the exchange may take
    auto v = pipe_bufs(ctx, z);
    for (const auto &b : exact_bufs(ctx, s.B, Bl, pull ? 1 : ctx->exchange_chunks)) v.push_back(b);
    v.push_back({&ctx->exch, pull ? 0 : std::max<uint64_t>(owned, 1) * sizeof(Row32)});
    v.push_back({&ctx->xcnt, slots ? Bl * 4 * W : 0});
    v.push_back({&ctx->xtotal, slots ? Bl * 4 : 0});
    v.push_back({&ctx->sortb, ctx->sort_classes ? sort_lists_scratch_bytes((uint32_t)Bl) : 0});
    return v;
}

size_t mp_pipe_bytes(tad_ctx *ctx, const tad_job *job, uint64_t global, uint64_t rows, uint64_t owned, bool slots)
{
    size_t b = 0;
    for (const auto &x : mp_pipe_bufs(ctx, job, global, rows, owned, slots)) b += x.second ? alloc_bytes(x.second) : 0;
    return b;
}

// A multi-GPU job under a memory budget.  Pass (v, P) holds the rows whose key hash has (h & (P-1)) == v on every rank at
// once; the owner rank is chosen by the top hash bits, so each pass is an ordinary multi-GPU job over the ranks' pass
// columns.  Every decision that changes which collectives a rank issues (the pass count, a split, the slot path, a cancel,
// a NOMEM verdict) is taken on all-gathered data, identically on every rank:
//   plan    one blocking all-gather of every rank's rows, pass capacity under its own budget, kept bytes and cancel flag;
//   counts  the first sweep counts every filtered row under (owner rank, residue): all-gathered, they give every rank's
//           input and owned rows of every pass for every P, so P is raised (pass 0 swept again, at most once) where some
//           rank would not fit, and the job fails with TAD_ERR_NOMEM on every rank where a 1/64 range does not fit one;
//   passes  run_pipeline at world_size > 1 over the pass columns, global_rows = the pass's total from the counts;
//   end     every pass ends with an 8-byte all-gather of {split, cancelled, fit stopped} (stop_word): a rank whose spill
//           scratch or result buffer does not fit, or whose fit stopped on the board, skips the rest of its pass but still
//           gets there, and then every rank splits the pass or stops.
// A rank stream job (TAD_FLAG_RANK_STREAM, DESIGN.md section 10, "Several GPUs") sweeps one round of its caller's blocks
// instead of its columns.  Its plan waits for its first block and carries its hint as its rows and its column set; the
// hint only seeds P0.  Its counts carry whether its first round's pass columns held all of pass (0, P0), its stop word,
// its input verdict, the rows its pass columns hold and the rows it delivered: P then comes from the delivered rows and
// the counts, and the pass columns are planned from the counts.  Every later round ends with an 8-byte all-gather of its
// stop word and verdict (its counts differ from its first round's), before the pipeline reads the pass.  Its rounds close
// on the same decisions on every rank, so every caller's tad_stream_end returns the same *again.
uint32_t run_passes_multi(tad_ctx *ctx, tad_job *job, uint64_t budget, PassOut &acc)
{
    cudaStream_t st = ctx->stream;
    const int W = ctx->cfg.world_size, me = ctx->cfg.rank, logW = log_world(ctx);
    const bool stream = job->rank_stream;
    set_progress(job, TAD_STATE_RUNNING, 0);
    StreamRound round{ctx, job};
    if (stream) round.first();
    const tad_columns &hc = job->cols;
    const uint64_t R = stream ? job->rows_hint : hc.rows;      // rows to plan for (a stream: its hint, 0 = unknown)
    const bool host = stream || (hc.mem != TAD_MEM_DEVICE && R > 0);
    Sweep sw(ctx, job, acc, host, budget, 0);
    const size_t stage_bytes = sw.stage_bytes();
    const size_t NC = (size_t)W * kMaxPasses;               // one rank's (owner, residue) counters
    // behind them, a stream's first round: pass 0 loaded, stop word, input verdict, pass-column rows held, rows delivered
    constexpr size_t kRoundWords = 5;
    const size_t NM = NC + kRoundWords;                      // one rank's counts message
    const size_t pcnt_bytes = (NM * (W + 1) + 1) * 8;        // mine, every rank's (all-gathered), the pass cursor

    // ---- plan ----------------------------------------------------------------------------------------------------------
    // what every pass keeps: pass columns of `n` rows, staging, counters, the ns_ignore list (and kFixedBytes)
    auto kept_bytes = [&](uint64_t n) {
        std::vector<std::pair<DevBuf *, size_t>> b = {{&ctx->stage, stage_bytes}, {&ctx->pcnt, pcnt_bytes},
                                                      {&ctx->ns_ignore, sw.ns ? job->ns_ignore.size() * 4 : 0}};
        for (int i = 0; i < 8; i++) b.push_back({&ctx->d_col[i], has_col(job, i) ? col_bytes(i, n) : 0});
        return workspace_after(ctx, b, true);
    };
    // rows one pass may hold on this rank: the largest n for which a pass whose input rows, owned rows and largest shard
    // are all n fits the budget (exact partition)
    const uint64_t cap = largest_fit(kMaxPassRows, budget, [&](uint64_t n) {
        const uint64_t g = n * (uint64_t)W;
        return kept_bytes(stream ? n : std::min(n, R)) + mp_pipe_bytes(ctx, job, g, n, n, false) +
               alloc_bytes(xbuf_bytes(ctx, g, n, false));
    });
    // rows the pass columns may hold: a table's shard; a stream's any count up to `cap` (its hint only seeds the plan)
    const uint64_t colcap = stream ? cap : std::min(cap, R);
    uint64_t mask = 0;               // the column set (a stream's agreed one: a rank whose first round is empty has none)
    for (int i = 0; i < 10; i++) mask |= has_col(job, i) ? 1ull << i : 0;

    // The budget applies from the plan on: until then the context may still hold the exported buffer of an earlier job,
    // larger than this budget, which only the plan all-gather lets it free.  No rank may fail on its own before it.
    ctx->limit = 0;
    ensure(ctx, ctx->small, tad_ctx::kSmallDevWords * 8);
    double gather_ms = 0;            // the small all-gathers' time: the ranks' skew (phase sync)
    // the exported buffer of an earlier job is freed for the plan: unmap the peers' buffers now, free ours once every rank
    // has (after the plan all-gather).  peers_mapped is the same on every rank.
    if (ctx->peers_mapped) CU(unmap_peers(ctx));
    ctx->x_agreed = 0;
    struct RankPlan {
        uint64_t rows, cap, budget, kept;
        bool cancel;
        uint64_t colcap, mask;
    } rk[kMaxRanks];
    memset(ctx->h_small, 0, tad_ctx::kGatherMax * 8);
    ctx->h_small[0] = R;
    ctx->h_small[1] = cap;
    ctx->h_small[2] = budget;
    ctx->h_small[3] = kept_bytes(stream ? 0 : colcap);   // a stream's pass columns are planned from its counts (need)
    ctx->h_small[4] = job->cancel.load() ? 1 : 0;
    ctx->h_small[5] = colcap;
    ctx->h_small[6] = mask;
    gather_ms += gather_small(ctx, tad_ctx::kGatherMax, true);
    for (int r = 0; r < W; r++) {
        const unsigned long long *w = ctx->h_small + tad_ctx::kGatherMax * (1 + r);
        rk[r] = RankPlan{w[0], w[1], w[2], w[3], w[4] != 0, w[5], w[6]};
    }
    free_buf(ctx, ctx->xbuf);
    ctx->limit = budget;
    ctx->peak = ctx->held;
    for (int r = 0; r < W; r++)
        if (rk[r].cancel) fail(TAD_ERR_CANCELLED, "job cancelled (rank %d)", r);
    if (stream) {
        int from = -1;
        for (int r = 0; r < W; r++) {
            if (!rk[r].mask) continue;
            if (from >= 0 && rk[r].mask != rk[from].mask)
                fail(TAD_ERR_INVALID_ARG, "invalid request: rank %d's blocks carry another set of columns than rank %d's",
                     r, from);
            if (from < 0) from = r;
        }
        if (!mask && from >= 0) adopt_columns(job, rk[from].mask);
        if (from >= 0) mask = rk[from].mask;
    }
    for (int r = 0; r < W; r++)
        if (rk[r].cap == 0)
            fail(TAD_ERR_NOMEM, "rank %d: a memory budget of %llu bytes does not hold one row of a pass", r,
                 (unsigned long long)rk[r].budget);
    // P from the rows rows_of(r): every rank's input and its share of the table within its capacity, with 1/8 head-room
    auto guess = [&](auto rows_of) {
        uint64_t total = 0;
        for (int r = 0; r < W; r++) total += rows_of(r);
        auto ok = [&](uint32_t p) {
            for (int r = 0; r < W; r++)
                if (std::max<uint64_t>(rows_of(r), (total + W - 1) / W) / p > rk[r].cap / 8 * 7) return false;
            return true;
        };
        uint32_t p = 1;
        while (p < (uint32_t)kMaxPasses && !ok(p)) p *= 2;
        return p;
    };
    uint32_t P = guess([&](int r) { return rk[r].rows; });
    const uint32_t P0 = P;
    // a stream's pass columns of n rows (at least kMinCols, so that a pass of no rows on a rank still has columns)
    constexpr uint64_t kMinCols = 2048;
    auto col_need = [&](uint64_t n) {
        size_t b = 0;
        for (int i = 0; i < 8; i++) b += mask >> i & 1 ? alloc_bytes(col_bytes(i, std::max(n, kMinCols))) : 0;
        return b;
    };

    // ---- pass columns and the sweep --------------------------------------------------------------------------------------
    // a stream's pass columns: from its hint (1M rows without one, kMinCols for an empty first round), grown while its
    // first round arrives (RoundGrowth)
    PassColumns pc(ctx, job);
    pc.size(!stream ? colcap : std::min(colcap, !round.have_pend ? kMinCols : R ? R / P + R / P / 8 + kMinCols : uint64_t(1) << 20));
    if (stage_bytes) ensure(ctx, ctx->stage, stage_bytes);
    ensure(ctx, ctx->pcnt, pcnt_bytes);
    ensure(ctx, ctx->stats, 64 * sizeof(uint32_t));
    unsigned long long *d_cnt = static_cast<unsigned long long *>(ctx->pcnt.p);
    unsigned long long *d_cursor = d_cnt + NM * (W + 1);
    sw.f = row_filter(ctx, job, sw.ns);
    sw.cnt = d_cnt;
    sw.cursor = d_cursor;
    sw.log_world = logW;
    bool count_only = false;         // the first round's pass columns could not grow inside the budget: it only counts
    RoundGrowth grow{ctx, pc, d_cursor, colcap, false, true, count_only};
    uint32_t sweeps = 0;
    bool unplanned = false;          // a later round brought host rows to a rank whose first round was empty (no staging)
    bool open = false;               // a streamed round is swept and its caller waits in tad_stream_end
    // the rows of pass (v, M) -> the pass columns, counted under (owner, residue)
    auto sweep = [&](uint32_t v, uint32_t M) {
        CU(cudaMemsetAsync(d_cnt, 0, NC * 8, st));
        CU(cudaMemsetAsync(d_cursor, 0, 8, st));
        sw.begin(host);
        if (!stream) {
            sw.feed(hc, 0, v, M, pc, false, nullptr);
        } else {
            grow.ub = 0;
            const uint64_t rows = round.run([&](const tad_columns &b, const tad_text_column *) {
                if (b.rows && b.mem != TAD_MEM_DEVICE && !sw.chunk) {
                    unplanned = true;
                    return st;
                }
                if (sweeps == 0 && !count_only) grow.room(b.rows);
                sw.feed(b, 0, v, M, pc, count_only, nullptr);
                return b.mem == TAD_MEM_DEVICE ? st : ctx->copy_stream;
            });
            if (sweeps == 0) job->round_rows = rows;
            open = true;
        }
        sw.end(false);
        sweeps++;
    };
    // a stream's input verdict in the agreed words: bit 32, a later round's counts differ from its first round's `mine`;
    // bits 40.., a block this rank refused (its error code, negated)
    auto input_word = [&](const uint64_t *mine) -> uint64_t {
        uint64_t w = 0;
        if (mine) {
            PinnedBlock hb = take_pinned(ctx, NC * 8);
            const cudaError_t e1 = cudaMemcpyAsync(hb.p, d_cnt, NC * 8, cudaMemcpyDeviceToHost, st);
            const cudaError_t e2 = cudaStreamSynchronize(st);
            const bool same = e1 == cudaSuccess && e2 == cudaSuccess && memcmp(hb.p, mine, NC * 8) == 0;
            give_pinned(ctx, hb);
            CU(e1);
            CU(e2);
            if (!same || unplanned) w |= 1ull << 32;
        }
        std::lock_guard<std::mutex> lk(job->mu);
        return w | (uint64_t)(uint32_t)(-job->in.err) << 40;
    };

    // ---- counts ----------------------------------------------------------------------------------------------------------
    sweep(0, P);
    std::vector<uint64_t> cnt(NC * W);       // [source rank][owner rank][residue]
    unsigned long long loaded_w[kMaxRanks], stop_w[kMaxRanks], input_w[kMaxRanks], pcap_w[kMaxRanks], rows_w[kMaxRanks];
    {
        CU(cudaMemcpyAsync(ctx->h_small + tad_ctx::kWPassCursor, d_cursor, 8, cudaMemcpyDeviceToHost, st));
        CU(cudaStreamSynchronize(st));
        ctx->h_small[0] = !count_only && ctx->h_small[tad_ctx::kWPassCursor] <= pc.cap;
        ctx->h_small[1] = stop_word(job, round.stopper);
        ctx->h_small[2] = stream ? input_word(nullptr) : 0;
        ctx->h_small[3] = pc.cap;
        ctx->h_small[4] = job->round_rows;
        CU(cudaMemcpyAsync(d_cnt + NC, ctx->h_small, kRoundWords * 8, cudaMemcpyHostToDevice, st));
        CU(cudaEventRecord(ctx->ev[0], st));
        if (nccl_allgather(&ctx->nccl, d_cnt, d_cnt + NM, NM * 8, st)) fail(TAD_ERR_NCCL, "%s", nccl_last_error());
        CU(cudaEventRecord(ctx->ev[1], st));
        PinnedBlock hb = take_pinned(ctx, NM * W * 8);
        const cudaError_t e1 = cudaMemcpyAsync(hb.p, d_cnt + NM, NM * W * 8, cudaMemcpyDeviceToHost, st);
        const cudaError_t e2 = cudaStreamSynchronize(st);
        if (e1 == cudaSuccess && e2 == cudaSuccess)
            for (int s = 0; s < W; s++) {
                const uint64_t *m = static_cast<const uint64_t *>(hb.p) + s * NM;
                memcpy(&cnt[s * NC], m, NC * 8);
                loaded_w[s] = m[NC];
                stop_w[s] = m[NC + 1];
                input_w[s] = m[NC + 2];
                pcap_w[s] = m[NC + 3];
                rows_w[s] = m[NC + 4];
            }
        give_pinned(ctx, hb);
        CU(e1);
        CU(e2);
        float ms = 0;
        CU(cudaEventElapsedTime(&ms, ctx->ev[0], ctx->ev[1]));
        gather_ms += ms;
    }
    if (stream) {
        agree_stop(stop_w, W);
        agree_input(job, input_w, W, me);
        count_only = false;          // later rounds split their pass into the pass columns
        // a wrong hint must not cost a round per surplus pass: plan from the rows the first round delivered, as exact hints
        // would have, at the price of that one round (loaded is then false unless P comes back to P0)
        P = std::min(P, guess([&](int r) { return rows_w[r]; }));
    }
    struct PassDims {
        uint64_t global = 0, max_rows = 0, rows[kMaxRanks] = {}, owned[kMaxRanks] = {};
    };
    auto dims = [&](uint32_t v, uint32_t M) {
        PassDims d;
        for (int s = 0; s < W; s++)
            for (int o = 0; o < W; o++)
                for (uint32_t j = v; j < (uint32_t)kMaxPasses; j += M) {
                    const uint64_t n = cnt[((size_t)s * W + o) * kMaxPasses + j];
                    d.rows[s] += n;
                    d.owned[o] += n;
                    d.global += n;
                }
        for (int s = 0; s < W; s++) d.max_rows = std::max(d.max_rows, d.rows[s]);
        return d;
    };
    // the exported buffer grows to the largest any pass of the plan needs and is never shrunk inside the job
    auto xbuf_of = [&](uint32_t M, bool slots) {
        size_t x = 0;
        for (uint32_t v = 0; v < M; v++) {
            const PassDims d = dims(v, M);
            if (d.global) x = std::max(x, xbuf_bytes(ctx, d.global, d.max_rows, slots));
        }
        return x;
    };
    // a rank's workspace in pass d; a stream's pass columns hold `cols` rows (the pass's rows when they are sized for it)
    auto need = [&](int r, const PassDims &d, bool slots, size_t x, uint64_t cols = 0) {
        return rk[r].kept + (stream ? col_need(std::max(cols, d.rows[r])) : 0) +
               mp_pipe_bytes(ctx, job, d.global, d.rows[r], d.owned[r], slots) + alloc_bytes(x);
    };
    int bad_r = 0;
    uint32_t bad_v = 0;
    // whether every pass of (., M) fits every rank
    auto fits_all = [&](uint32_t M, bool slots) {
        const size_t x = xbuf_of(M, slots);
        for (uint32_t v = 0; v < M; v++) {
            const PassDims d = dims(v, M);
            if (!d.global) continue;
            for (int r = 0; r < W; r++)
                if (d.rows[r] > rk[r].colcap || d.owned[r] > kMaxPassRows ||
                    need(r, d, slots, x) > rk[r].budget) {
                    bad_r = r;
                    bad_v = v;
                    return false;
                }
        }
        return true;
    };
    while (P < (uint32_t)kMaxPasses && !fits_all(P, false)) P *= 2;
    auto too_big = [&](int r, uint32_t v, uint32_t M) {
        const PassDims d = dims(v, M);
        fail(TAD_ERR_NOMEM, "rank %d: one 1/%u hash range of the table (%llu rows in, %llu owned) needs %zu bytes of device "
             "workspace; its memory budget is %llu bytes", r, M, (unsigned long long)d.rows[r], (unsigned long long)d.owned[r],
             need(r, d, false, xbuf_of(M, false)), (unsigned long long)rk[r].budget);
    };
    if (!fits_all(P, false)) too_big(bad_r, bad_v, P);
    // the slot path where its exported buffer fits next to the workspace of every pass on every rank
    const bool slots = ctx->peer_pull && ctx->optimistic && fits_all(P, true);
    const size_t xplan = xbuf_of(P, slots);
    bool loaded = P == P0;           // pass (0, P) is in the pass columns already (a stream's: on every rank, in columns
                                     // that fit its plan)
    for (int r = 0; r < W && stream && loaded; r++)
        loaded = loaded_w[r] && need(r, dims(0, P), slots, xplan, pcap_w[r]) <= rk[r].budget;
    // a stream's round stays open until the ranks know whether another round follows: one does while a queued pass has
    // rows (a loaded pass 0 may still split)
    auto finish_round = [&](bool more) {
        if (!open) return;
        close_round(job, more);
        open = false;
    };
    uint64_t counted = 0;
    for (uint64_t n : cnt) counted += n;
    if (!loaded) finish_round(counted > 0);

    // ---- passes ----------------------------------------------------------------------------------------------------------
    auto run_one = [&](uint32_t v, uint32_t M, const PassList &rest, PassOut &o) {
        const PassDims d = dims(v, M);
        if (!loaded) {                // the round the previous pass was swept in closes once that pass has run
            bool more = d.global > 0;
            for (const auto &e : rest) more = more || dims(e.first, e.second).global > 0;
            finish_round(more);
        }
        if (!d.global) {              // the same on every rank: no collective
            loaded = false;
            return false;
        }
        if (!loaded && stream) {
            // columns too small, or too large for the plan: sized for the pass, the earlier passes' buffers freed first
            if (d.rows[me] > pc.cap || pc.cap < kMinCols || need(me, d, slots, xplan, pc.cap) > budget) {
                free_pass_buffers(ctx);
                pc.drop();
                pc.size(std::max(d.rows[me], kMinCols));
            }
            sweep(v, M);
            // the round's verdict, agreed before the pipeline reads the pass: a cancel, a stop read off the board, a
            // refused block, or counts that differ from the first round's (the pass columns then disagree with the
            // agreed sizes the pipeline's exchange is planned from)
            ctx->h_small[0] = stop_word(job, round.stopper) | input_word(&cnt[me * NC]);
            gather_ms += gather_small(ctx, 1, true);
            agree_stop(ctx->h_small + 1, W);
            agree_input(job, ctx->h_small + 1, W, me);
        } else if (!loaded) {
            sweep(v, M);
        }
        loaded = false;
        // the buffers of earlier passes go where this pass's growth would pass the budget
        const size_t xgrow = alloc_bytes(xplan) > ctx->xbuf.cap ? alloc_bytes(xplan) - ctx->xbuf.cap : 0;
        if (workspace_after(ctx, mp_pipe_bufs(ctx, job, d.global, d.rows[me], d.owned[me], slots), false) + xgrow > budget)
            free_pass_buffers(ctx);
        bool split_here = false;
        try {
            const AgreedPass ap{d.global, d.max_rows};
            run_pipeline(ctx, job, pc.as_input(d.rows[me]), false, !slots, o, &ap);
        } catch (const PassSplit &) {
            CU(cudaStreamSynchronize(st));
            split_here = true;
        }
        // ---- the agreed end of the pass: {split, cancelled, fit stopped} of every rank ----
        ctx->h_small[0] = (split_here ? 1u : 0u) | stop_word(job, o.fit_stop >= 0 ? o.fit_stop : round.stopper);
        gather_ms += gather_small(ctx, 1, true);
        int split_r = -1;
        for (int r = W - 1; r >= 0; r--)
            if (ctx->h_small[1 + r] & 1) split_r = r;
        const bool stop = any_stop(ctx->h_small + 1, W);
        if (!stop && split_r < 0) return false;
        give_pinned(ctx, o.block);
        agree_stop(ctx->h_small + 1, W);
        if (M >= (uint32_t)kMaxPasses)
            fail(TAD_ERR_NOMEM, "rank %d: the oversized-bucket scratch or result buffer of a 1/%d hash range of the "
                 "table (%llu rows owned) does not fit its memory budget of %llu bytes", split_r, kMaxPasses,
                 (unsigned long long)d.owned[split_r], (unsigned long long)rk[split_r].budget);
        return true;
    };
    const uint32_t passes = run_pass_queue(ctx, job, P, acc, run_one);
    finish_round(false);
    acc.phase_ms[TAD_PHASE_SYNC] += gather_ms;
    acc.device_ms += gather_ms;
    return passes;
}

// `reserve`: a job run while an ARIMA fit is parked (interleave), with the fit-sharing reserve as its budget.
void run_job(tad_ctx *ctx, tad_job *job, uint64_t reserve)
{
    CU(cudaSetDevice(ctx->cfg.device));
    // a loopback rank (ranks as contexts of one process) waits for its turn on the device; released by worker_main
    if (nccl_job_begin(&ctx->nccl)) fail(TAD_ERR_NCCL, "%s", nccl_last_error());
    // several GPUs: a job cancelled in the queue runs to its first agreed point (the plan all-gather under a budget, else
    // the verdict), and its stop is written now, so that the peers' fits stop at once
    if (ctx->cfg.world_size > 1) {
        if (!ctx->boards_shared) share_boards(ctx);
        std::lock_guard<std::mutex> lk(job->mu);
        job->started = true;
        if (job->cancel.load()) post_stop(ctx, job->ordinal);
    } else if (job->cancel.load()) {
        fail(TAD_ERR_CANCELLED, "job cancelled");
    }
    const uint64_t multi_budget = ctx->cfg.world_size > 1 ? ctx->budget.load() : 0;
    const tad_columns &hc = job->cols;     // a streamed job's first push writes it: not read here for streams
    const uint64_t R = job->stream ? 0 : hc.rows;
    ctx->limit = 0;
    const uint64_t host_budget = reserve ? store_share(ctx) : store_trim(ctx);      // the job's one read of the host budget
    // fit sharing: a single-GPU ARIMA job, submitted or streamed with TAD_FLAG_SHARE, plans in the budget less the reserve,
    // and its fit yields
    const bool may_share = !job->stream || (job->spec.flags & TAD_FLAG_SHARE);
    job->share = !reserve && may_share && ctx->cfg.world_size == 1 && job->spec.algo == TAD_ALGO_ARIMA ? ctx->fit_share.load() : 0;
    // an ARIMA job run in a yield fits beside the parked fit (TAD_FLAG_FIT_BESIDE): it is a sharing job whose budget is
    // the reserve and whose own reserve, where the jobs run in its yields go, is half of it
    if (reserve && job->spec.algo == TAD_ALGO_ARIMA) job->share = reserve / 2;
    // lending (TAD_FLAG_LEND): a single-GPU streamed job run in its own turn, not in a yield, while sharing is on; it plans
    // in the budget less the reserve, where the jobs run in its lends go
    job->lend = !reserve && job->stream && (job->spec.flags & TAD_FLAG_LEND) && ctx->cfg.world_size == 1
                    ? ctx->fit_share.load() : 0;
    // ---- plan (single GPU): one pass as today when it fits the budget, else hash-range passes ----------------------
    uint64_t budget = 0;
    bool force_exact = false, split = false;
    const uint64_t set = reserve ? reserve : ctx->budget.load();
    auto context_budget = [&]() -> uint64_t {
        if (set) return set;
        size_t free_b = 0, total_b = 0;
        CU(cudaMemGetInfo(&free_b, &total_b));
        return free_b + ctx->held > kBudgetHeadroom ? free_b + ctx->held - kBudgetHeadroom : 0;
    };
    const uint64_t held_back = std::max(job->share, job->lend);      // the reserve of a job that yields, lends or both
    auto less_reserve = [&](uint64_t b) {
        if (!held_back) return b;
        if (b < held_back + kBudgetFloor)
            fail(TAD_ERR_NOMEM, "a memory budget of %llu bytes less the fit-sharing reserve of %llu bytes is below the "
                 "64 MiB floor", (unsigned long long)b, (unsigned long long)held_back);
        return b - held_back;
    };
    if (job->stream) {
        // streamed input always runs through the pass columns (one pass when it fits), under the budget (a rank stream
        // job's: run_passes_multi applies it once the plan has freed the exported buffer)
        set_progress(job, TAD_STATE_RUNNING, 0);
        budget = less_reserve(context_budget());
        ctx->limit = budget;
        free_workspace(ctx);
        split = true;
    } else if (multi_budget) {
        budget = multi_budget;          // run_passes_multi applies it once the plan has freed the exported buffer
        free_workspace(ctx);
    } else if (ctx->cfg.world_size == 1 && R > 0) {
        budget = less_reserve(context_budget());
        PipeShape s = one_gpu_shape(ctx, job, R, true);
        s.host = hc.mem != TAD_MEM_DEVICE ? &hc : nullptr;
        auto bufs = pipe_bufs(ctx, pipe_sizes(s));
        if (workspace_after(ctx, bufs, true) > budget) {
            s.optimistic = false;
            force_exact = true;
            bufs = pipe_bufs(ctx, pipe_sizes(s));
            split = workspace_after(ctx, bufs, true) > budget;
        }
        if (set || force_exact || job->share) {
            ctx->limit = budget;
            if (split || workspace_after(ctx, bufs, false) > budget) free_workspace(ctx);
        }
    }
    ctx->peak = ctx->held;
    PassOut acc;
    uint32_t passes = 1;
    const bool multi = multi_budget || job->rank_stream;
    if (multi) {
        passes = run_passes_multi(ctx, job, budget, acc);
    } else if (!split) {
        set_passes(job, 0, 1);
        try {
            run_pipeline(ctx, job, hc, true, force_exact, acc);
            set_passes(job, 1, 1);
        } catch (const PassSplit &) {          // thrown only under a budget
            CU(cudaStreamSynchronize(ctx->stream));
            acc = PassOut{};
            const tad_progress none{};
            set_passes(job, 0, 1, &none);
            split = true;
        }
    }
    if (split && !multi) passes = run_passes(ctx, job, budget, host_budget, reserve != 0, acc);
    publish_rows(job, acc.block, acc.out_rows);
    ctx->limit = 0;
    {
        std::lock_guard<std::mutex> lk(job->mu);
        tad_status &s = job->st;
        s.rows_in = job->stream ? job->round_rows : R;
        s.rows_kept = acc.kept;
        s.rows_owned = acc.owned;
        s.points = acc.points;
        s.series = acc.series;
        s.result_rows = acc.out_rows;
        s.spill_rows = acc.spill_rows;
        s.gpu_launches = acc.launches;
        s.device_ms = acc.device_ms;
        for (int i = 0; i < TAD_NPHASES; i++) s.phase_ms[i] = acc.phase_ms[i];
        s.total_ms = now_ms() - job->t_submit;
        s.completed_stages = kTotalStages;
        s.state = TAD_STATE_COMPLETED;
        job->passes = passes;
        job->peak_workspace = ctx->peak;
        job->peak_host = ctx->store_peak;
        job->cv.notify_all();     // last touch of `job` by the worker (tad_release may free it now)
    }
}

// Runs `job` and reports a failure on it.  `reserve` (interleave): false when the job failed with TAD_ERR_NOMEM inside
// the reserve; it is then SCHEDULED again with no progress, is not run beside a fit again, and waits for its turn.  A
// streamed one first has its round in progress closed with again = 1 (discard_round) and starts again from its first
// round, with empty dictionaries.
bool run_one(tad_ctx *ctx, tad_job *job, uint64_t reserve)
{
    JobFail f;
    try {
        run_job(ctx, job, reserve);
        return true;
    } catch (const JobFail &e) {
        f = e;
    }
    // nothing of this job may still be reading the caller's columns once it is reported FAILED
    cudaStreamSynchronize(ctx->copy_stream);
    cudaStreamSynchronize(ctx->stream);
    cudaStreamSynchronize(ctx->d2h_stream);
    cudaGetLastError();
    TextKeys::release(ctx);
    if (reserve && f.code == TAD_ERR_NOMEM && !job->cancel.load()) {
        try {
            if (job->stream) discard_round(job);
            std::lock_guard<std::mutex> lk(job->mu);
            job->no_interleave = true;
            job->st.state = TAD_STATE_SCHEDULED;
            job->st.completed_stages = 0;
            job->prog = tad_progress{};
            job->round_rows = job->stored_rows = 0;
            return false;
        } catch (const JobFail &e) {       // cancelled, or a bad block, while the round was taken to its end
            f = e;
        }
    }
    std::lock_guard<std::mutex> lk(job->mu);
    job->st.state = TAD_STATE_FAILED;
    job->st.error = f.code;
    snprintf(job->st.err_msg, sizeof(job->st.err_msg), "%s", f.msg);
    job->st.total_ms = now_ms() - job->t_submit;
    job->cv.notify_all();
    return true;
}

void worker_main(tad_ctx *ctx)
{
    if (ctx->numa.ok) sched_setaffinity(0, sizeof(ctx->numa.cpus), &ctx->numa.cpus);      // this thread only
    cudaSetDevice(ctx->cfg.device);
    for (;;) {
        tad_job *job = nullptr;
        {
            std::unique_lock<std::mutex> lk(ctx->mu);
            ctx->cv.wait(lk, [&] { return ctx->stop || !ctx->queue.empty(); });
            if (ctx->queue.empty()) return;       // stop requested and drained
            job = ctx->queue.front();
            ctx->queue.pop_front();
        }
        run_one(ctx, job, 0);
        nccl_job_end(&ctx->nccl);      // a loopback rank's streams are idle: its peers may take the device
    }
}

int validate(const tad_job_spec *spec, const tad_columns *cols, char *msg, size_t n)
{
    if (spec->algo != TAD_ALGO_EWMA && spec->algo != TAD_ALGO_ARIMA && spec->algo != TAD_ALGO_DBSCAN) {
        // controller.go:527-529
        snprintf(msg, n, "invalid request: Throughput Anomaly Detector algorithm type should be 'EWMA' or 'ARIMA' or 'DBSCAN'");
        return TAD_ERR_INVALID_ARG;
    }
    if (spec->reducer != TAD_REDUCE_MAX && spec->reducer != TAD_REDUCE_SUM) {
        snprintf(msg, n, "invalid request: reducer should be max or sum");
        return TAD_ERR_INVALID_ARG;
    }
    if (spec->start_time && spec->end_time && spec->end_time <= spec->start_time) {
        // controller.go:535-539
        snprintf(msg, n, "invalid request: EndInterval should be after StartInterval");
        return TAD_ERR_INVALID_ARG;
    }
    if (cols->rows && (!cols->flow_end || !cols->value)) {
        snprintf(msg, n, "invalid request: flow_end and value columns are required");
        return TAD_ERR_INVALID_ARG;
    }
    if (cols->rows && spec->start_time && !cols->flow_start) {
        // flowStartSeconds >= start filters on the flow_start KEY column; a job whose key has none (the external / svc
        // aggregated modes, anomaly_detection.py:568-571) applies that bound on the host, where the column lives
        snprintf(msg, n, "invalid request: start_time needs the flow_start column");
        return TAD_ERR_INVALID_ARG;
    }
    if (cols->rows >= (1ull << 32) - 1) {
        snprintf(msg, n, "invalid request: at most 2^32-2 rows per GPU");
        return TAD_ERR_INVALID_ARG;
    }
    if (cols->mem != TAD_MEM_HOST && cols->mem != TAD_MEM_DEVICE) {
        snprintf(msg, n, "invalid request: bad column memory kind");
        return TAD_ERR_INVALID_ARG;
    }
    if (spec->n_ns_ignore && !spec->ns_ignore) {
        snprintf(msg, n, "invalid request: ns_ignore is NULL");
        return TAD_ERR_INVALID_ARG;
    }
    return TAD_OK;
}

// Validates and enqueues a job (tad_submit, tad_submit_stream).  An invalid job is returned FAILED, like the controller
// (controller.go:505-514): illegal arguments are terminal, never retried.
int submit_job(tad_ctx *ctx, tad_job *job, const tad_job_spec *spec, const tad_columns *cols, tad_job **out)
{
    job->ctx = ctx;
    job->spec = *spec;
    job->spec.id[sizeof(job->spec.id) - 1] = 0;
    job->cols = *cols;
    job->t_submit = now_ms();
    job->st.total_stages = kTotalStages;
    *out = job;
    char msg[200];
    int rc = validate(spec, cols, msg, sizeof(msg));
    if (rc == TAD_OK && job->stream && ctx->cfg.world_size > 1 && !job->rank_stream) {
        snprintf(msg, sizeof(msg), "streamed input runs on a single GPU only, or on every rank with TAD_FLAG_RANK_STREAM");
        rc = TAD_ERR_UNSUPPORTED;
    }
    if (rc != TAD_OK) {
        job->st.state = TAD_STATE_FAILED;
        job->st.error = rc;
        snprintf(job->st.err_msg, sizeof(job->st.err_msg), "error in creating AnomalyDetector: %s", msg);
        return rc;
    }
    if (spec->n_ns_ignore) job->ns_ignore.assign(spec->ns_ignore, spec->ns_ignore + spec->n_ns_ignore);
    job->spec.ns_ignore = nullptr;
    job->st.state = TAD_STATE_SCHEDULED;
    {
        std::lock_guard<std::mutex> lk(ctx->mu);
        if (ctx->stop) {
            job->st.state = TAD_STATE_FAILED;
            job->st.error = TAD_ERR_STATE;
            snprintf(job->st.err_msg, sizeof(job->st.err_msg), "context is shutting down");
            return TAD_ERR_STATE;
        }
        job->ordinal = ++ctx->job_seq;      // jobs are queued in the same order on every rank: so are the ordinals
        ctx->queue.push_back(job);
    }
    ctx->cv.notify_one();
    return TAD_OK;
}

bool finished(const tad_job *job) { return job->st.state == TAD_STATE_COMPLETED || job->st.state == TAD_STATE_FAILED; }

// Fails a streamed job from the caller's side (a bad block) and waits until the worker has reported it FAILED.
int stream_abort(tad_job *job, std::unique_lock<std::mutex> &lk, int code, const char *msg)
{
    if (!job->in.err) {
        job->in.err = code;
        snprintf(job->in.msg, sizeof(job->in.msg), "%s", msg);
    }
    job->cv.notify_all();
    while (!finished(job)) job->cv.wait_for(lk, std::chrono::milliseconds(5));
    return code;
}

// A rank stream job cancelled on this rank, or whose engine read a peer's stop off its board: its caller's push and end
// calls return TAD_ERR_CANCELLED without waiting for its peers, once the engine reads none of its blocks (a block handed
// over but not taken is withdrawn).
bool rank_halted(const tad_job *job) { return job->rank_stream && (job->cancel.load() || job->peer_stop.load()); }

int rank_cancelled(tad_job *job, std::unique_lock<std::mutex> &lk)
{
    job->in.has_blk = false;
    while (!finished(job) && job->in.released < job->in.taken) job->cv.wait_for(lk, std::chrono::milliseconds(5));
    return TAD_ERR_CANCELLED;
}

// Whether a push or end call is legal now: TAD_ERR_STATE on a job without streamed input or after its input is complete;
// TAD_ERR_CANCELLED (once the job is FAILED) after tad_cancel; the job's error once it has failed.
int stream_gate(tad_job *job, std::unique_lock<std::mutex> &lk)
{
    if (!job->stream || job->in.input_done) return TAD_ERR_STATE;
    if (rank_halted(job)) return rank_cancelled(job, lk);
    if (job->cancel.load()) {
        while (!finished(job)) job->cv.wait_for(lk, std::chrono::milliseconds(5));
        return TAD_ERR_CANCELLED;
    }
    if (finished(job)) return job->st.error ? job->st.error : TAD_ERR_STATE;
    return TAD_OK;
}

// A streamed block: host or device memory, fewer than 2^32 rows, flow_end and value, and the first block's column set,
// text slots included.  A text slot: host memory, its u32 column NULL, one mark per 32 rows from 0, not decreasing, none
// past the column's end.  Namespace slots: all text or all u32, text only with the ignore list as names and names only
// with text.
int check_block(const tad_job *job, const tad_columns *b, const tad_text_column *const *txt, char *msg, size_t n)
{
    static const char *kSlot[4] = {"src_ip", "dst_ip", "src_ns", "dst_ns"};
    for (int t = 0; t < 4; t++) {
        const tad_text_column *x = txt[t];
        if (!x) continue;
        if (b->mem != TAD_MEM_HOST) {
            snprintf(msg, n, "invalid request: text key columns are accepted in host blocks only");
            return TAD_ERR_INVALID_ARG;
        }
        if (col_ptr(*b, t < 2 ? t : t + 6)) {
            snprintf(msg, n, "invalid request: a slot given as text must have its u32 column NULL");
            return TAD_ERR_INVALID_ARG;
        }
        const uint64_t nseg = (b->rows + 31) / 32;
        if ((x->nbytes && !x->bytes) || (nseg && !x->marks) || (nseg && x->marks[0] != 0)) {
            snprintf(msg, n, "invalid request: a text column needs its bytes and one mark per 32 rows, the first 0");
            return TAD_ERR_INVALID_ARG;
        }
        for (uint64_t s = 0; s < nseg; s++)
            if (x->marks[s] > x->nbytes || (s && x->marks[s] < x->marks[s - 1])) {
                snprintf(msg, n, "invalid request: the marks of a text column decrease or pass its end");
                return TAD_ERR_INVALID_ARG;
            }
    }
    if ((txt[2] || txt[3]) && (b->src_ns || b->dst_ns)) {
        snprintf(msg, n, "invalid request: a streamed block gives one namespace column as text and the other as u32 ids");
        return TAD_ERR_INVALID_ARG;
    }
    if ((txt[2] || txt[3]) && job->spec.n_ns_ignore) {
        snprintf(msg, n, "invalid request: namespace text needs the ignore list as names (tad_submit_stream_filtered_ns), "
                 "not as ids");
        return TAD_ERR_INVALID_ARG;
    }
    if (job->ns_names && (b->src_ns || b->dst_ns)) {
        snprintf(msg, n, "invalid request: an ignore list of names needs the namespace columns as text, not as u32 ids");
        return TAD_ERR_INVALID_ARG;
    }
    if (job->in.pushed > 0)
        for (int t = 0; t < 4; t++)
            if (job->text[t] != (txt[t] != nullptr)) {
                snprintf(msg, n, "invalid request: a streamed block gives %s as %s, the job's first block did not",
                         kSlot[t], txt[t] ? "text" : "u32");
                return TAD_ERR_INVALID_ARG;
            }
    if (b->mem != TAD_MEM_HOST && b->mem != TAD_MEM_DEVICE) {
        snprintf(msg, n, "invalid request: bad column memory kind");
        return TAD_ERR_INVALID_ARG;
    }
    if (b->rows >= (1ull << 32)) {
        snprintf(msg, n, "invalid request: a streamed block has fewer than 2^32 rows");
        return TAD_ERR_INVALID_ARG;
    }
    if (!b->flow_end || !b->value) {
        snprintf(msg, n, "invalid request: flow_end and value columns are required");
        return TAD_ERR_INVALID_ARG;
    }
    if (job->in.pushed == 0) {
        for (int t = 0; t < 2; t++)
            if (job->name_op[t] != TAD_NAME_ANY && !txt[t]) {
                snprintf(msg, n, "invalid request: a row predicate on %s, which the first block does not give as text",
                         t ? "dst_ip" : "src_ip");
                return TAD_ERR_INVALID_ARG;
            }
        if (job->proto_eq >= 0 && (!b->proto || (!txt[0] && !txt[1]))) {
            snprintf(msg, n, "invalid request: proto_eq needs the proto column and a text key slot");
            return TAD_ERR_INVALID_ARG;
        }
        if (job->spec.start_time && !b->flow_start) {
            snprintf(msg, n, "invalid request: start_time needs the flow_start column");
            return TAD_ERR_INVALID_ARG;
        }
        return TAD_OK;
    }
    for (int i = 0; i < 10; i++)
        if ((col_ptr(job->cols, i) != nullptr) != (col_ptr(*b, i) != nullptr)) {
            snprintf(msg, n, "invalid request: a streamed block carries another set of columns than the job's first block");
            return TAD_ERR_INVALID_ARG;
        }
    return TAD_OK;
}

}  // namespace

// =============================================================================================
// C ABI
// =============================================================================================
extern "C" {

int tad_abi_version(void) { return TAD_ABI_VERSION; }

int tad_get_unique_id(void *out, size_t bytes)
{
    if (!out || bytes < 128) return TAD_ERR_INVALID_ARG;
    return nccl_get_unique_id(out, bytes) == 0 ? TAD_OK : TAD_ERR_NCCL;
}

const char *tad_strerror(int err)
{
    const int i = -err;
    if (i < 0 || i > 8) return "unknown error";
    return kErrNames[i];
}

int tad_init(const tad_config *cfg, tad_ctx **out)
{
    if (!cfg || !out) return TAD_ERR_INVALID_ARG;
    if (cfg->world_size < 1 || cfg->rank < 0 || cfg->rank >= cfg->world_size) return TAD_ERR_INVALID_ARG;
    if (cfg->world_size > kMaxRanks || (cfg->world_size & (cfg->world_size - 1))) return TAD_ERR_INVALID_ARG;   // 1, 2, 4, 8
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
        cudaGetLastError();
        fprintf(stderr, "theia_tad: no CUDA device is available; this library has no CPU fallback\n");
        return TAD_ERR_CUDA;
    }
    if (cfg->device < 0 || cfg->device >= ndev) return TAD_ERR_INVALID_ARG;
    if (cudaSetDevice(cfg->device) != cudaSuccess) return TAD_ERR_CUDA;
    tad_ctx *ctx = new tad_ctx();
    ctx->cfg = *cfg;
    ctx->cfg.nccl_unique_id = nullptr;
    if (const char *e = getenv("TAD_DEBUG_LOGB")) ctx->debug_logb = atoi(e);
    if (const char *e = getenv("TAD_DEBUG_TEXT_MASK")) ctx->text_mask = strtoull(e, nullptr, 16);
    if (const char *e = getenv("TAD_DEBUG_NO_GROW")) ctx->debug_no_grow = atoi(e) != 0;
    if (const char *e = getenv("TAD_GROUP_TARGET")) ctx->debug_target = atoi(e);
    cudaDeviceGetAttribute(&ctx->num_sms, cudaDevAttrMultiProcessorCount, cfg->device);
    ctx->numa = numa_of_device(cfg->device);
    NumaScope numa_scope(ctx->numa);
    bool ok = cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking) == cudaSuccess;
    ok = ok && cudaStreamCreateWithFlags(&ctx->copy_stream, cudaStreamNonBlocking) == cudaSuccess;
    ok = ok && cudaStreamCreateWithFlags(&ctx->d2h_stream, cudaStreamNonBlocking) == cudaSuccess;
    for (int i = 0; ok && i < 2; i++) ok = cudaEventCreateWithFlags(&ctx->ost_ev[i], cudaEventDisableTiming) == cudaSuccess;
    for (int i = 0; ok && i < 2; i++) ok = cudaEventCreateWithFlags(&ctx->cnt_ev[i], cudaEventDisableTiming) == cudaSuccess;
    for (int i = 0; ok && i < kMaxChunks; i++) ok = cudaEventCreateWithFlags(&ctx->chunk_ev[i], cudaEventDisableTiming) == cudaSuccess;
    ok = ok && cudaEventCreateWithFlags(&ctx->start_ev, cudaEventDisableTiming) == cudaSuccess;
    for (int i = 0; ok && i < 2; i++) ok = cudaEventCreateWithFlags(&ctx->stage_ev[i], cudaEventDisableTiming) == cudaSuccess;
    for (int i = 0; ok && i < 2; i++) ok = cudaEventCreateWithFlags(&ctx->blk_ev[i], cudaEventDisableTiming) == cudaSuccess;
    for (int i = 0; ok && i <= kMaxXChunks; i++) ok = cudaEventCreateWithFlags(&ctx->x_ev[i], cudaEventDisableTiming) == cudaSuccess;
    if (const char *e = getenv("TAD_OPTIMISTIC")) ctx->optimistic = atoi(e);
    // defaults = the fastest measured configuration per world size (DESIGN.md section 6): peer pull everywhere, the exact fallback
    // pulled as well, capacity-class lists sorted by bucket from 4 ranks on (locality of the small remote reads)
    ctx->peer_pull = 1;
    ctx->exact_pull = 1;
    ctx->sort_classes = cfg->world_size >= 4 ? 1 : 0;
    if (const char *e = getenv("TAD_PEER_PULL")) ctx->peer_pull = atoi(e);
    if (const char *e = getenv("TAD_EXACT_PULL")) ctx->exact_pull = atoi(e);
    if (const char *e = getenv("TAD_SORT_CLASSES")) ctx->sort_classes = atoi(e);
    if (const char *e = getenv("TAD_SLOT_BUDGET_GB")) ctx->x_budget = (size_t)strtoull(e, nullptr, 10) << 30;
    if (const char *e = getenv("TAD_EXCHANGE_MIN_ROWS")) ctx->exchange_min_rows = strtoull(e, nullptr, 10);
    if (getenv("TAD_EXCHANGE_CHUNKS")) ctx->exchange_chunks_forced = true;
    if (const char *e = getenv("TAD_EXCHANGE_CHUNKS")) ctx->exchange_chunks = atoi(e) < 1 ? 1 : (atoi(e) > kMaxXChunks ? kMaxXChunks : atoi(e));
    for (int i = 0; ok && i < kMaxEvents; i++) ok = cudaEventCreate(&ctx->ev[i]) == cudaSuccess;
    for (int i = 0; ok && i < 2 * kMaxEvents; i++) ok = cudaEventCreate(&ctx->ev_alt[i / kMaxEvents][i % kMaxEvents]) == cudaSuccess;
    ok = ok && cudaHostAlloc((void **)&ctx->h_stats, 64 * sizeof(uint32_t), cudaHostAllocDefault) == cudaSuccess;
    ok = ok && cudaHostAlloc((void **)&ctx->h_small, tad_ctx::kSmallWords * sizeof(unsigned long long), cudaHostAllocDefault) == cudaSuccess;
    ok = ok && cudaHostAlloc((void **)&ctx->h_chunk, 2 * kMaxPasses * sizeof(uint32_t), cudaHostAllocDefault) == cudaSuccess;
    ok = ok && cudaHostAlloc((void **)&ctx->h_fit, sizeof(tad_ctx::FitPinned), cudaHostAllocDefault) == cudaSuccess;
    if (ok) *ctx->h_fit = tad_ctx::FitPinned{};
    for (int i = 0; ok && i < 2; i++) ok = cudaEventCreateWithFlags(&ctx->fit_ev[i], cudaEventDisableTiming) == cudaSuccess;
    ok = ok && cudaEventCreateWithFlags(&ctx->fits_ev, cudaEventDisableTiming) == cudaSuccess;
    if (ok && cfg->world_size > 1) {
        // the stop board: allocated here, once, and mapped by the peers in the first job (share_boards)
        ok = cudaMalloc((void **)&ctx->board, 4 * kMaxRanks) == cudaSuccess;
        ok = ok && cudaMemset(ctx->board, 0, 4 * kMaxRanks) == cudaSuccess;
        ok = ok && cudaStreamCreateWithFlags(&ctx->board_stream, cudaStreamNonBlocking) == cudaSuccess;
        ok = ok && cudaHostAlloc((void **)&ctx->h_board, 16 * sizeof(uint32_t), cudaHostAllocDefault) == cudaSuccess;
        if (ok) {
            memset(ctx->h_board, 0, 16 * sizeof(uint32_t));
            ctx->peer_board[cfg->rank] = ctx->board;
        }
    }
    if (!ok) {
        tad_shutdown(ctx);      // releases whatever was created
        return TAD_ERR_CUDA;
    }
    if (cfg->world_size > 1) {
        ctx->nccl.streams[0] = ctx->stream;
        ctx->nccl.streams[1] = ctx->copy_stream;
        ctx->nccl.streams[2] = ctx->d2h_stream;
        int rc = nccl_comm_init(&ctx->nccl, cfg->world_size, cfg->rank, cfg->nccl_unique_id, cfg->nccl_unique_id_bytes);
        if (rc != 0) {
            tad_shutdown(ctx);
            return TAD_ERR_NCCL;
        }
    }
    ctx->worker = std::thread(worker_main, ctx);
    *out = ctx;
    return TAD_OK;
}

void tad_shutdown(tad_ctx *ctx)
{
    if (!ctx) return;
    {
        std::lock_guard<std::mutex> lk(ctx->mu);
        ctx->stop = true;
    }
    ctx->stopping.store(1);
    ctx->cv.notify_all();
    if (ctx->worker.joinable()) ctx->worker.join();
    cudaSetDevice(ctx->cfg.device);
    if ((ctx->peers_mapped || ctx->boards_shared) && ctx->nccl.comm && ctx->small.p && ctx->stream) {
        // an exported buffer or board must outlive every peer's mapping of it: unmap, meet the peers, only then free
        unmap_peers(ctx);
        for (int r = 0; r < ctx->cfg.world_size; r++) {
            if (r != ctx->cfg.rank && ctx->peer_board[r]) nccl_ipc_unmap(&ctx->nccl, ctx->peer_board[r]);
            ctx->peer_board[r] = nullptr;
        }
        if (peer_barrier(ctx) == 0) cudaStreamSynchronize(ctx->stream);
    }
    nccl_comm_destroy(&ctx->nccl);
    drop_buf(ctx, ctx->xbuf);
    free_bufs(ctx);
    for (auto &b : ctx->pinned_pool) cudaFreeHost(b.p);
    for (auto &b : ctx->store_slabs) cudaFreeHost(b.p);
    if (ctx->h_chunk) cudaFreeHost(ctx->h_chunk);
    if (ctx->h_stats) cudaFreeHost(ctx->h_stats);
    if (ctx->h_small) cudaFreeHost(ctx->h_small);
    if (ctx->h_fit) cudaFreeHost(ctx->h_fit);
    if (ctx->h_board) cudaFreeHost(ctx->h_board);
    if (ctx->board) cudaFree(ctx->board);
    if (ctx->board_stream) cudaStreamDestroy(ctx->board_stream);
    for (int i = 0; i < 2; i++)
        if (ctx->fit_ev[i]) cudaEventDestroy(ctx->fit_ev[i]);
    if (ctx->fits_ev) cudaEventDestroy(ctx->fits_ev);
    for (int i = 0; i < kMaxEvents; i++) {
        if (ctx->ev[i]) cudaEventDestroy(ctx->ev[i]);
        for (auto &alt : ctx->ev_alt)
            if (alt[i]) cudaEventDestroy(alt[i]);
    }
    for (int i = 0; i < kMaxChunks; i++)
        if (ctx->chunk_ev[i]) cudaEventDestroy(ctx->chunk_ev[i]);
    if (ctx->start_ev) cudaEventDestroy(ctx->start_ev);
    for (int i = 0; i < 2; i++)
        if (ctx->stage_ev[i]) cudaEventDestroy(ctx->stage_ev[i]);
    for (int i = 0; i < 2; i++)
        if (ctx->blk_ev[i]) cudaEventDestroy(ctx->blk_ev[i]);
    for (int i = 0; i < 2; i++) {
        if (ctx->ost_ev[i]) cudaEventDestroy(ctx->ost_ev[i]);
        if (ctx->cnt_ev[i]) cudaEventDestroy(ctx->cnt_ev[i]);
    }
    for (int i = 0; i <= kMaxXChunks; i++)
        if (ctx->x_ev[i]) cudaEventDestroy(ctx->x_ev[i]);
    if (ctx->copy_stream) cudaStreamDestroy(ctx->copy_stream);
    if (ctx->d2h_stream) cudaStreamDestroy(ctx->d2h_stream);
    if (ctx->stream) cudaStreamDestroy(ctx->stream);
    delete ctx;
}

int tad_alloc_columns(tad_ctx *ctx, uint64_t capacity, int32_t mem, tad_columns *cols)
{
    if (!ctx || !cols || (mem != TAD_MEM_HOST && mem != TAD_MEM_DEVICE)) return TAD_ERR_INVALID_ARG;
    memset(cols, 0, sizeof(*cols));
    cols->capacity = capacity;
    cols->mem = mem;
    if (cudaSetDevice(ctx->cfg.device) != cudaSuccess) return TAD_ERR_CUDA;
    NumaScope numa_scope(ctx->numa);
    void **slots[8] = {(void **)&cols->src_ip, (void **)&cols->dst_ip, (void **)&cols->src_port, (void **)&cols->dst_port,
                       (void **)&cols->proto, (void **)&cols->flow_start, (void **)&cols->flow_end, (void **)&cols->value};
    for (int i = 0; i < 8; i++) {
        const size_t bytes = ((col_bytes(i, capacity ? capacity : 1)) + 255) & ~size_t(255);
        cudaError_t e = mem == TAD_MEM_HOST ? cudaHostAlloc(slots[i], bytes, cudaHostAllocDefault) : cudaMalloc(slots[i], bytes);
        if (e != cudaSuccess) {
            cudaGetLastError();
            tad_free_columns(ctx, cols);
            return TAD_ERR_NOMEM;
        }
    }
    return TAD_OK;
}

int tad_alloc_ns_columns(tad_ctx *ctx, tad_columns *cols)
{
    if (!ctx || !cols || !cols->capacity) return TAD_ERR_INVALID_ARG;
    if (cudaSetDevice(ctx->cfg.device) != cudaSuccess) return TAD_ERR_CUDA;
    NumaScope numa_scope(ctx->numa);
    void **slots[2] = {(void **)&cols->src_ns, (void **)&cols->dst_ns};
    for (int i = 0; i < 2; i++) {
        if (*slots[i]) continue;
        const size_t bytes = (cols->capacity * 4 + 255) & ~size_t(255);
        cudaError_t e = cols->mem == TAD_MEM_HOST ? cudaHostAlloc(slots[i], bytes, cudaHostAllocDefault) : cudaMalloc(slots[i], bytes);
        if (e != cudaSuccess) {
            cudaGetLastError();
            return TAD_ERR_NOMEM;
        }
    }
    return TAD_OK;
}

int tad_free_columns(tad_ctx *ctx, tad_columns *cols)
{
    if (!ctx || !cols) return TAD_ERR_INVALID_ARG;
    cudaSetDevice(ctx->cfg.device);
    for (int i = 0; i < 10; i++) {
        void *p = col_ptr(*cols, i);
        if (!p) continue;
        if (cols->mem == TAD_MEM_HOST) cudaFreeHost(p); else cudaFree(p);
    }
    memset(cols, 0, sizeof(*cols));
    return TAD_OK;
}

int tad_submit(tad_ctx *ctx, const tad_job_spec *spec, const tad_columns *cols, tad_job **out)
{
    if (!ctx || !spec || !cols || !out) return TAD_ERR_INVALID_ARG;
    return submit_job(ctx, new tad_job(), spec, cols, out);
}

int tad_submit_stream(tad_ctx *ctx, const tad_job_spec *spec, uint64_t rows_hint, tad_job **out)
{
    if (!ctx || !spec || !out) return TAD_ERR_INVALID_ARG;
    tad_job *job = new tad_job();
    job->stream = true;
    job->rank_stream = (spec->flags & TAD_FLAG_RANK_STREAM) && ctx->cfg.world_size > 1;
    job->rows_hint = rows_hint;
    tad_columns none{};
    return submit_job(ctx, job, spec, &none, out);
}

int tad_submit_stream_filtered(tad_ctx *ctx, const tad_job_spec *spec, uint64_t rows_hint, const tad_stream_filter *filter,
                               tad_job **out)
{
    if (!filter) return tad_submit_stream(ctx, spec, rows_hint, out);
    const tad_stream_filter_ns f{*filter, 0, nullptr, nullptr};
    return tad_submit_stream_filtered_ns(ctx, spec, rows_hint, &f, out);
}

int tad_submit_stream_filtered_ns(tad_ctx *ctx, const tad_job_spec *spec, uint64_t rows_hint,
                                  const tad_stream_filter_ns *filter_ns, tad_job **out)
{
    if (!filter_ns) return tad_submit_stream(ctx, spec, rows_hint, out);
    if (!ctx || !spec || !out) return TAD_ERR_INVALID_ARG;
    const tad_stream_filter *filter = &filter_ns->rows;
    const char *bad = nullptr;
    for (int t = 0; t < 2 && !bad; t++) {
        const int op = filter->op[t];
        const uint32_t m = filter->pattern_len[t];
        if (op < TAD_NAME_ANY || op > TAD_NAME_ICONTAINS) bad = "a row predicate op is not a TAD_NAME_* value";
        else if (m && !filter->pattern[t]) bad = "a row predicate pattern is NULL with a nonzero length";
        else if (op == TAD_NAME_ICONTAINS)
            for (uint32_t k = 0; k < m && !bad; k++)
                if (filter->pattern[t][k] >= 0x80) bad = "an ICONTAINS pattern holds a byte >= 0x80 (ASCII only)";
    }
    if (!bad && (filter->proto_eq < -1 || filter->proto_eq > 255)) bad = "proto_eq is outside -1..255";
    const uint32_t nn = filter_ns->n_ns_ignore;
    const uint64_t *off = filter_ns->ns_ignore_offsets;
    if (!bad && nn && (!off || !filter_ns->ns_ignore_bytes)) bad = "the ignore list's bytes or offsets are NULL";
    if (!bad && nn && spec->n_ns_ignore) bad = "the ignore list is given both as names and as ids";
    if (!bad && nn > kNsMaxNames) bad = "the ignore list holds more than 1024 names";
    if (!bad && nn && off[0] != 0) bad = "the ignore list's offsets do not start at 0";
    for (uint32_t k = 0; k < nn && !bad; k++)
        if (off[k + 1] < off[k]) bad = "the ignore list's offsets decrease";
    if (!bad && nn && off[nn] > kNsMaxBytes) bad = "the ignore list's names hold more than 32 KiB";
    tad_job *job = new tad_job();
    job->stream = true;
    job->rows_hint = rows_hint;
    if (bad) {                   // returned FAILED, as submit_job returns an invalid job
        job->ctx = ctx;
        job->spec = *spec;
        job->st.total_stages = kTotalStages;
        job->st.state = TAD_STATE_FAILED;
        job->st.error = TAD_ERR_INVALID_ARG;
        snprintf(job->st.err_msg, sizeof(job->st.err_msg), "error in creating AnomalyDetector: invalid request: %s", bad);
        *out = job;
        return TAD_ERR_INVALID_ARG;
    }
    for (int t = 0; t < 2; t++) {
        job->name_op[t] = filter->op[t];
        // only EQ and ICONTAINS read a pattern
        if (filter->op[t] == TAD_NAME_EQ || filter->op[t] == TAD_NAME_ICONTAINS)
            job->name_pat[t].assign(filter->pattern[t], filter->pattern[t] + filter->pattern_len[t]);
    }
    job->proto_eq = filter->proto_eq;
    if (nn) {                    // the namespace text slots stage kNsListed for a listed name: the row filter drops it
        job->ns_image = ns_list_image(filter_ns->ns_ignore_bytes, off, nn, ctx->text_mask);
        job->ns_names = nn;
        job->ns_ignore.assign(1, kNsListed);
    }
    tad_columns none{};
    return submit_job(ctx, job, spec, &none, out);
}

int tad_stream_push(tad_job *job, const tad_columns *block)
{
    return tad_stream_push_text_ns(job, block, nullptr, nullptr, nullptr, nullptr);
}

int tad_stream_push_text(tad_job *job, const tad_columns *block, const tad_text_column *src_ip, const tad_text_column *dst_ip)
{
    return tad_stream_push_text_ns(job, block, src_ip, dst_ip, nullptr, nullptr);
}

int tad_stream_push_text_ns(tad_job *job, const tad_columns *block, const tad_text_column *src_ip,
                            const tad_text_column *dst_ip, const tad_text_column *src_ns, const tad_text_column *dst_ns)
{
    if (!job || !block) return TAD_ERR_INVALID_ARG;
    if ((src_ip || dst_ip || src_ns || dst_ns) && !job->stream) return TAD_ERR_UNSUPPORTED;
    std::unique_lock<std::mutex> lk(job->mu);
    int rc = stream_gate(job, lk);
    if (rc != TAD_OK) return rc;
    if ((src_ip || dst_ip || src_ns || dst_ns) && job->rank_stream) {   // the ranks would need a dictionary they agree on
        if (!job->in.err) {
            job->in.err = TAD_ERR_UNSUPPORTED;
            snprintf(job->in.msg, sizeof(job->in.msg), "text key columns are not supported on a job streamed to several GPUs");
            job->cv.notify_all();
        }
        return TAD_ERR_UNSUPPORTED;
    }
    char msg[200];
    const tad_text_column *txt[4] = {src_ip, dst_ip, src_ns, dst_ns};
    rc = check_block(job, block, txt, msg, sizeof(msg));
    if (rc != TAD_OK) return stream_abort(job, lk, rc, msg);
    if (job->in.pushed == 0) {                         // the column set of the job
        job->cols = *block;
        for (int t = 0; t < 4; t++) job->text[t] = txt[t] != nullptr;
    }

    // one block of look-ahead: hand this one over once the worker has taken the previous one, then return once the
    // engine no longer reads the previous one
    while (job->in.has_blk && !finished(job) && !rank_halted(job)) job->cv.wait_for(lk, std::chrono::milliseconds(5));
    if (rank_halted(job)) return rank_cancelled(job, lk);
    if (finished(job)) return job->st.error;
    job->in.blk = *block;
    for (int t = 0; t < 4; t++) job->in.txt[t] = txt[t] ? *txt[t] : tad_text_column{};
    job->in.has_blk = true;
    const uint64_t k = job->in.pushed++;
    job->cv.notify_all();
    while (job->in.released < k && !finished(job) && !rank_halted(job)) job->cv.wait_for(lk, std::chrono::milliseconds(5));
    if (rank_halted(job)) return rank_cancelled(job, lk);
    return finished(job) ? job->st.error : TAD_OK;
}

int tad_stream_end(tad_job *job, int32_t *again)
{
    if (!job) return TAD_ERR_INVALID_ARG;
    std::unique_lock<std::mutex> lk(job->mu);
    int rc = stream_gate(job, lk);
    if (rc != TAD_OK) return rc;
    while (job->in.has_blk && !finished(job) && !rank_halted(job)) job->cv.wait_for(lk, std::chrono::milliseconds(5));
    if (rank_halted(job)) return rank_cancelled(job, lk);
    if (finished(job)) return job->st.error;
    job->in.end_req = true;
    job->cv.notify_all();
    while (!job->in.round_done && !finished(job) && !rank_halted(job)) job->cv.wait_for(lk, std::chrono::milliseconds(5));
    if (rank_halted(job)) return rank_cancelled(job, lk);
    if (!job->in.round_done) return job->st.error;
    job->in.round_done = false;
    job->in.input_done = !job->in.again;
    if (again) *again = job->in.again ? 1 : 0;
    return TAD_OK;
}

int tad_poll(tad_job *job, tad_status *status)
{
    if (!job || !status) return TAD_ERR_INVALID_ARG;
    std::lock_guard<std::mutex> lk(job->mu);
    *status = job->st;
    return TAD_OK;
}

int tad_wait(tad_job *job, int64_t timeout_ms, tad_status *status)
{
    if (!job) return TAD_ERR_INVALID_ARG;
    std::unique_lock<std::mutex> lk(job->mu);
    auto done = [&] { return job->st.state == TAD_STATE_COMPLETED || job->st.state == TAD_STATE_FAILED; };
    if (timeout_ms < 0) {
        while (!done()) job->cv.wait_for(lk, std::chrono::milliseconds(50));
    } else {
        const double deadline = now_ms() + (double)timeout_ms;
        while (!done() && now_ms() < deadline) job->cv.wait_for(lk, std::chrono::milliseconds(1));
    }
    if (status) *status = job->st;
    return TAD_OK;
}

int tad_result(tad_job *job, tad_rows *rows)
{
    if (!job || !rows) return TAD_ERR_INVALID_ARG;
    std::lock_guard<std::mutex> lk(job->mu);
    if (job->st.state != TAD_STATE_COMPLETED) return TAD_ERR_STATE;
    *rows = job->rows;
    return TAD_OK;
}

int tad_cancel(tad_job *job)
{
    if (!job) return TAD_ERR_INVALID_ARG;
    std::lock_guard<std::mutex> lk(job->mu);
    job->cancel.store(1);
    stop_running(job);
    job->cv.notify_all();        // a worker waiting for streamed input
    return TAD_OK;
}

int tad_job_progress(tad_job *job, tad_progress *p)
{
    if (!job || !p) return TAD_ERR_INVALID_ARG;
    std::lock_guard<std::mutex> lk(job->mu);
    *p = job->prog;
    return TAD_OK;
}

int tad_set_memory_budget(tad_ctx *ctx, uint64_t bytes)
{
    if (!ctx) return TAD_ERR_INVALID_ARG;
    if (bytes && bytes < kBudgetFloor) return TAD_ERR_INVALID_ARG;
    ctx->budget.store(bytes);
    return TAD_OK;
}

int tad_set_fit_sharing(tad_ctx *ctx, uint64_t reserve_bytes)
{
    if (!ctx) return TAD_ERR_INVALID_ARG;
    if (ctx->cfg.world_size > 1) return TAD_ERR_UNSUPPORTED;
    if (reserve_bytes && reserve_bytes < kBudgetFloor) return TAD_ERR_INVALID_ARG;
    ctx->fit_share.store(reserve_bytes);
    return TAD_OK;
}

int tad_job_yields(tad_job *job, uint32_t *yields, double *parked_ms)
{
    if (!job) return TAD_ERR_INVALID_ARG;
    std::lock_guard<std::mutex> lk(job->mu);
    if (job->st.state != TAD_STATE_COMPLETED || job->spec.algo != TAD_ALGO_ARIMA) return TAD_ERR_STATE;
    if (yields) *yields = job->yields;
    if (parked_ms) *parked_ms = job->parked_ms;
    return TAD_OK;
}

int tad_job_lent(tad_job *job, uint32_t *jobs_run, double *lent_ms)
{
    if (!job || !jobs_run || !lent_ms) return TAD_ERR_INVALID_ARG;
    std::lock_guard<std::mutex> lk(job->mu);
    if (job->st.state != TAD_STATE_COMPLETED || !job->stream) return TAD_ERR_STATE;
    *jobs_run = job->lent_jobs;
    *lent_ms = job->lent_ms;
    return TAD_OK;
}

int tad_job_memory(tad_job *job, uint32_t *passes, uint64_t *peak_workspace_bytes)
{
    if (!job) return TAD_ERR_INVALID_ARG;
    std::lock_guard<std::mutex> lk(job->mu);
    if (job->st.state != TAD_STATE_COMPLETED) return TAD_ERR_STATE;
    if (passes) *passes = job->passes;
    if (peak_workspace_bytes) *peak_workspace_bytes = job->peak_workspace;
    return TAD_OK;
}

int tad_job_names(tad_job *job, int32_t slot, const uint8_t **bytes, const uint64_t **offsets, uint32_t *count)
{
    if (!job || slot < 0 || slot > 1 || !bytes || !offsets || !count) return TAD_ERR_INVALID_ARG;
    std::lock_guard<std::mutex> lk(job->mu);
    if (job->st.state != TAD_STATE_COMPLETED || !job->text[slot]) return TAD_ERR_STATE;
    *bytes = job->names[slot].data();
    *offsets = job->names_off[slot].data();
    *count = (uint32_t)(job->names_off[slot].size() - 1);
    return TAD_OK;
}

int tad_set_host_budget(tad_ctx *ctx, uint64_t bytes)
{
    if (!ctx) return TAD_ERR_INVALID_ARG;
    if (ctx->cfg.world_size > 1) return TAD_ERR_UNSUPPORTED;
    if (bytes && bytes < kBudgetFloor) return TAD_ERR_INVALID_ARG;
    ctx->host_budget.store(bytes);
    return TAD_OK;
}

int tad_job_host_memory(tad_job *job, uint64_t *stored_rows, uint64_t *peak_host_bytes)
{
    if (!job) return TAD_ERR_INVALID_ARG;
    std::lock_guard<std::mutex> lk(job->mu);
    if (job->st.state != TAD_STATE_COMPLETED) return TAD_ERR_STATE;
    if (stored_rows) *stored_rows = job->stored_rows;
    if (peak_host_bytes) *peak_host_bytes = job->peak_host;
    return TAD_OK;
}

int tad_release(tad_job *job)
{
    if (!job) return TAD_ERR_INVALID_ARG;
    {
        std::unique_lock<std::mutex> lk(job->mu);
        const int s = job->st.state;
        if (s == TAD_STATE_SCHEDULED || s == TAD_STATE_RUNNING) {
            job->cancel.store(1);
            stop_running(job);
            job->cv.notify_all();
            while (!(job->st.state == TAD_STATE_COMPLETED || job->st.state == TAD_STATE_FAILED))
                job->cv.wait_for(lk, std::chrono::milliseconds(1));
        }
    }
    give_pinned(job->ctx, job->result_block);
    delete job;
    return TAD_OK;
}

}  // extern "C"
