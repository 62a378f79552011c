// Shared definitions of the TAD engine kernels (sm_90a).
//
// Data layout in HBM (DESIGN.md section 3):
//   input    : structure-of-arrays flow columns (tad_columns), 29 B/row for the full key
//   part[]   : hash-partitioned rows, 32 B each (Row32) = exactly one DRAM sector, so a
//              fully random scatter has no write amplification
//   csr_v/t  : per-series, time-sorted, duplicate-reduced values (u64) / flowEndSeconds (u32)
//   entries  : one 32 B SeriesEntry per connection, written IN PLACE over the dead part[]
//              region of its bucket (a bucket is fully staged in shared memory before its
//              entries are written)
//   EWMA writes csr_v/t and entries for spilled buckets only: the group kernel scores the others.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace tad {

struct __align__(32) Row32 {
    uint64_t a;       // src_ip << 32 | dst_ip
    uint64_t b;       // flow_start << 32 | src_port << 16 | dst_port
    uint64_t value;   // throughput
    uint32_t t;       // flow_end
    uint32_t proto;   // bits 0-7 protocolIdentifier; bits 8-31: the 24 key-hash bits below the bucket bits (hash tag)
};
static_assert(sizeof(Row32) == 32, "Row32 must be one 32-byte sector");

struct __align__(32) SeriesEntry {
    uint64_t a, b;
    uint32_t proto;
    uint32_t n;       // points after the stage-A reduce
    uint32_t off;     // first point in csr_v / csr_t
    uint32_t pad;
};
static_assert(sizeof(SeriesEntry) == 32, "SeriesEntry aliases a Row32 slot");

struct ColPtrs {
    const uint32_t *src_ip, *dst_ip, *flow_start, *flow_end;
    const uint16_t *src_port, *dst_port;
    const uint8_t *proto;
    const uint64_t *value;
    const uint32_t *src_ns, *dst_ns;
};

struct RowFilter {
    uint32_t start_time, end_time;   // 0 = unbounded
    uint32_t n_ns_ignore;
    const uint32_t *ns_ignore;       // device pointer
};

// A bucket's rows may arrive as several segments: one per source rank after the multi-GPU exchange
// (one segment, the local partition buffer itself, on a single GPU).  Segment r holds the rows of
// this rank's bucket range in bucket order; off[r] is the exclusive row offset of every bucket in it.
constexpr int kMaxSeg = 32;          // 8 source ranks x 4 exchange chunks
struct SegDesc {
    const Row32 *base[kMaxSeg];
    const uint32_t *off[kMaxSeg];   // stride == 0: exclusive row offsets (B_local + 1); stride != 0 && nseg > 1: row COUNTS (B_local)
    int nseg;
    uint32_t stride;      // != 0: fixed-capacity slots (optimistic partition): local bucket b of segment s starts at
                          // base[s] + (b_lo + b) * stride.  One segment on a single GPU (the slot holds min(count, stride)
                          // rows, the rest sits in the overflow list); one segment PER SOURCE RANK on several GPUs, where
                          // base[s] is rank s's partition buffer mapped into this process (CUDA IPC) and the rows are
                          // pulled over NVLink -- no exchange step, no receive buffer.
    uint32_t b_lo;        // first global bucket of this rank's range (0 on a single GPU)
};

// rows of local bucket `bkt` that segment `sg` holds, and where they start (n_total: the bucket's total, single segment only)
__host__ __device__ __forceinline__ void seg_span(const SegDesc &seg, int sg, uint32_t bkt, uint32_t n_total, uint32_t &first,
                                                  uint32_t &count)
{
    if (seg.stride) {
        first = (seg.b_lo + bkt) * seg.stride;
        count = seg.nseg == 1 ? n_total : seg.off[sg][bkt];
    } else {
        first = seg.off[sg][bkt];
        count = seg.off[sg][bkt + 1] - first;
    }
}

struct OutCols {
    uint32_t *src_ip, *dst_ip, *flow_start, *flow_end;
    uint16_t *src_port, *dst_port;
    uint8_t *proto, *anomaly;
    double *stddev, *algo_calc, *throughput;
};

__host__ __device__ __forceinline__ uint64_t mix64(uint64_t x)
{
    x ^= x >> 33; x *= 0xff51afd7ed558ccdULL; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ULL; x ^= x >> 33;
    return x;
}

// 64-bit hash of the 136-bit connection key.  Top bits select the bucket (and, across
// GPUs, the owner rank); the next bits select the shared-memory hash-table slot.
__host__ __device__ __forceinline__ uint64_t key_hash(uint64_t a, uint64_t b, uint32_t proto)
{
    return mix64(a ^ mix64(b + 0x9e3779b97f4a7c15ULL * (uint64_t)(proto + 1u)));
}

// Shared-memory capacity classes of the group kernel, smallest first: a bucket of 0 < n <= kGroupCap rows goes to the
// first class whose capacity holds it.  Every class runs four rows per thread except the 768-row class, which runs six:
// seven CTAs of 192 threads would leave the fused instance 40 registers (it spills), seven of 128 leave it 72.  `ctas` is
// the CTAs per SM the fused (EWMA) instance is built for (its __launch_bounds__); a static_assert on each class's
// shared-memory footprint keeps it reachable.  The bucket scan, the class lists, the ST_NCLS* counters and the group
// launchers all derive from this table.
struct GroupClass { int cap, threads, ctas; };
constexpr int kGroupClasses = 7;
__host__ __device__ constexpr GroupClass group_class(int c)
{
    constexpr GroupClass t[kGroupClasses] = {{512, 128, 10}, {768, 128, 7}, {1024, 256, 5}, {1280, 320, 4},
                                             {1536, 384, 3}, {2048, 512, 2}, {4096, 1024, 1}};
    return t[c];
}

// device scalars the host reads back between phases
enum {
    ST_KEPT = 0,        // rows that passed the stage-A filters
    ST_NBIG,            // buckets larger than the shared-memory capacity
    ST_BIGROWS,         // rows in those buckets
    ST_MAXBUCKET,
    ST_SERIES,          // total series
    ST_POINTS,          // total points after the reduce
    ST_OUTCOUNT,        // result rows produced (may exceed capacity -> rerun)
    ST_NCLS0,           // [ST_NCLS0, +kGroupClasses): buckets per shared-memory capacity class (group_class)
    ST_OVF = ST_NCLS0 + kGroupClasses,           // optimistic partition: rows that did not fit their bucket's fixed-capacity slot
    ST_LOCALKEPT,       // multi-GPU optimistic partition: rows of THIS rank that passed the filters (ST_KEPT = rows owned);
                        // must follow ST_OVF: the two travel in one 8-byte all-gather
    ST_GSERIES,         // EWMA: series / points of the buckets the group kernel scored in place (ST_SERIES / ST_POINTS
    ST_GPOINTS,         // then count the spilled buckets only); adjacent: zeroed together before every scoring attempt
    ST_COUNT
};
// ARIMA fit launch, outside the ST_COUNT readback: [ST_FITS, +2) the fit counters (FitPart's fits_total, fits_done), which
// the worker copies back while the fit kernel runs, [ST_FITS + 2] the kernel's cancel word, and [ST_FITS + 3] scratch of
// a fit beside a yielded one
constexpr int ST_FITS = 32;

constexpr int kGroupCap = group_class(kGroupClasses - 1).cap;   // rows a bucket may hold to take the shared-memory path
constexpr int kGroupTarget = 768;     // mean rows per bucket pick_logb aims for


// sbase[] layout (written by the series scan): [0, B] exclusive scan of series per bucket (sbase[B] = S), followed by the
// bucket hint table: hint[j] = bucket of series 32 * j.  A detector finds the bucket of series i with one hint load and a
// short forward walk (32 series span a handful of buckets) instead of a log2(B)-deep chain of dependent loads.
constexpr uint32_t kHintStride = 32;
__host__ __device__ __forceinline__ size_t sbase_words(uint32_t B, uint64_t max_series) { return (size_t)B + 1 + max_series / kHintStride + 2; }
#ifdef __CUDACC__
__device__ __forceinline__ uint32_t find_bucket(const uint32_t *__restrict__ sbase, uint32_t B, uint32_t i)
{
    uint32_t b = sbase[B + 1 + i / kHintStride];      // bucket of series (i rounded down to a multiple of 32) <= bucket of i
    while (sbase[b + 1] <= i) b++;                     // terminates: sbase[B] = S > i
    return b;
}
#endif

}  // namespace tad
