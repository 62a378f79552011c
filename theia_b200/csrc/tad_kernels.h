// Launchers of the TAD engine kernels (implemented in tad_kernels.cu, tad_spill.cu, tad_arima.cu).
#pragma once
#include "tad_common.cuh"

namespace tad {

cudaError_t launch_hist(cudaStream_t st, const ColPtrs &c, uint64_t R, const RowFilter &f, int logB, uint32_t *hist);
// slot_cap == 0: exact mode, cursor[] holds absolute row cursors (from the bucket scan).
// slot_cap  > 0: optimistic mode, cursor[] counts arrivals from zero, bucket b owns part[b * slot_cap ...); rows past the
//                slot go to ovf[] (ovf_count may exceed ovf_cap: the caller then falls back to the exact partition).
cudaError_t launch_scatter(cudaStream_t st, const ColPtrs &c, uint64_t R, const RowFilter &f, int logB, uint32_t *cursor,
                           Row32 *part, uint32_t slot_cap = 0, Row32 *ovf = nullptr, uint32_t ovf_cap = 0,
                           uint32_t *ovf_count = nullptr);
// Hash-range passes: the rows of `c` that pass the stage-A filters and whose key hash has (h & pass_mask) == pass_val
// are appended at out[*cursor ...) (rows past `cap` are dropped, *cursor still counts them); counts[kMaxPasses] gains
// the filtered rows of every low-hash-bit residue.  Null key columns of `out` are skipped (they read as 0 anyway).
// The cursor and counts are 64-bit: one sweep over a streamed round may hold more than 2^32 rows.
// `mark` (here and in launch_residue_pack): 1 / 2 = a row whose src_ip / dst_ip id has bit 31 set (a failed text
// predicate, tad_text.h) is dropped as well; 0 = no such bit.
// `log_world` 1..3 (2, 4 or 8 ranks; mark must be 0): counts[2^log_world x kMaxPasses] gains the filtered rows under
// (owner rank, residue) instead, owner = the top log_world bits of the key hash, as the multi-GPU pipeline assigns owners.
constexpr int kMaxPasses = 64;
struct PassCols {
    uint32_t *src_ip, *dst_ip, *flow_start, *flow_end;
    uint16_t *src_port, *dst_port;
    uint8_t *proto;
    uint64_t *value;
};
cudaError_t launch_pass_split(cudaStream_t st, const ColPtrs &c, uint64_t R, const RowFilter &f, uint32_t pass_mask,
                              uint32_t pass_val, const PassCols &out, uint32_t cap, unsigned long long *cursor,
                              unsigned long long *counts, int mark = 0, int log_world = 0);
// Host row store: the rows of `c` that pass the stage-A filters, packed as Row32 records without the hash tag, grouped
// by low-hash-bit residue (residue 0 first) into out[0, rows kept).  chunk[kMaxPasses] (u32, zeroed here) receives the
// rows of every residue and totals[kMaxPasses] (null: skipped) gains them.  R <= the max_rows the scratch was sized for;
// three launches.
size_t residue_pack_scratch_bytes(uint64_t max_rows);
cudaError_t launch_residue_pack(cudaStream_t st, const ColPtrs &c, uint64_t R, const RowFilter &f, void *scratch,
                                size_t scratch_bytes, uint32_t *chunk, unsigned long long *totals, Row32 *out, int mark = 0);
// Stored rows in[0, n) -> out columns at rows [at, at + n); null key columns are skipped.  One launch.
cudaError_t launch_store_unpack(cudaStream_t st, const Row32 *in, uint64_t n, const PassCols &out, uint64_t at);
cudaError_t launch_bucket_scan(cudaStream_t st, const uint32_t *hist, uint32_t *offsets, uint32_t *cursor, uint32_t B,
                               uint32_t cap, uint32_t *big_list, uint32_t *big_base, uint32_t *cls_list /* kGroupClasses x B or null */,
                               uint32_t *stats, void *scan_sync, uint32_t epoch);
size_t scan_sync_bytes();   // zero-initialised once; epoch must be > 0 and differ between launches
// csr_p != nullptr: also rank every series by value and write the permutation (value rank -> time
// index) the DBSCAN detector sweeps over.
// `offsets` are the (virtual, contiguous) bucket offsets used for entries / csr arrays; the rows
// themselves are read through `seg`.
cudaError_t launch_group(cudaStream_t st, const SegDesc &seg, SeriesEntry *entries, const uint32_t *offsets, uint32_t B,
                         const uint32_t *cls_list, const uint32_t n_cls[kGroupClasses], uint64_t *csr_v, uint32_t *csr_t,
                         uint32_t *csr_p, uint32_t *nsb, uint32_t *npb, int reducer, int *launches);
// EWMA scored inside the group kernel: every bucket of the class lists is grouped, time-sorted, reduced and scored in
// shared memory, and its flagged points (every point with emit_all) go straight to out[0, out_cap); rows past out_cap are
// counted, not written.  stats[ST_OUTCOUNT] gains the result rows, stats[ST_GSERIES] / [ST_GPOINTS] the series and points.
// Writes no series entries, per-series arrays or nsb / npb, and never writes over the bucket rows it reads, so a relaunch
// with the three counters zeroed gives the same rows.
struct GroupScore {
    OutCols out;
    uint32_t out_cap;
    uint32_t *stats;
    int emit_all;
};
cudaError_t launch_group_ewma(cudaStream_t st, const SegDesc &seg, const uint32_t *offsets, uint32_t B, const uint32_t *cls_list,
                              const uint32_t n_cls[kGroupClasses], int reducer, const GroupScore &score, int *launches);
cudaError_t launch_series_scan(cudaStream_t st, const uint32_t *nsb, const uint32_t *npb, uint32_t *sbase, uint32_t B,
                               uint32_t *stats, void *scan_sync, uint32_t epoch);
cudaError_t launch_detect_ewma(cudaStream_t st, const SeriesEntry *entries, const uint32_t *offsets, const uint32_t *sbase, uint32_t B,
                               uint32_t S, const uint64_t *csr_v, const uint32_t *csr_t, const OutCols &out,
                               uint32_t out_cap, uint32_t *stats, int emit_all);
cudaError_t launch_detect_dbscan(cudaStream_t st, const SeriesEntry *entries, const uint32_t *offsets, const uint32_t *sbase,
                                 uint32_t B, uint32_t S, const uint64_t *csr_v, const uint32_t *csr_t, const uint32_t *csr_p,
                                 uint32_t *scratch_pc, uint8_t *scratch_flag, const OutCols &out, uint32_t out_cap,
                                 uint32_t *stats, int emit_all);

// ARIMA (tad_arima.cu): the per-prefix ARIMA(1,1,1) MLE fits of a pass's series into pred[], then launch_detect_arima
// scores / flags / compacts (one launch, rerun alone when the result grows).
// FitPart: one job's fit as a launcher takes it.  y / pred: one double per point slot; lam: one double per series.
// fits_total, fits_done, cancel: the words of the fit (u32: one fit per point, fewer than 2^32 points per pass).
//   fits_total gains the prefix fits of the series (Box-Cox) and fits_done, the word after it (the worker copies both
//   back at once), the fits finished.  The fit kernel reads the cancel word in every round; nonzero = every warp leaves
//   at its next round and drops the fits in flight, so pred[] is then incomplete.
// resume (2 S + 2 u32): the fit can yield (null: it cannot).  A cancel word of 2 makes every warp leave like a cancel,
//   after it has written its series' resume point and the fits it dropped there ([2i], [2i + 1]); [2S] gains the fits
//   dropped, [2S + 1] the dropped fits a resume launch has finished again (both zeroed by the caller).
struct FitPart {
    const SeriesEntry *entries;
    const uint32_t *offsets, *sbase;
    uint32_t B, S;
    double *y, *lam, *pred;
    uint32_t *cancel;
    uint32_t *fits_done, *resume;
    uint32_t *fits_total;
};
// launch_arima_boxcox: y = the Box-Cox transformed series, lam, and fits_total; with resume, pred[] marked as not fitted.
// launch_arima_fit: launch_arima_boxcox, then the fit kernel (two launches).  board (multi-GPU jobs, with resume null):
//   the fit stops on the ranks' stop board instead of the cancel word -- 8 u32 in this rank's device memory, one per rank
//   (the rest 0); every warp leaves at its next round once a word equals `ordinal`.
// launch_arima_resume: fits what a yield left (the fits dropped in flight and those never started) into the same pred[]
//   and counters, so the forecasts and counts are those of one launch.
// Fitting beside a yielded fit (TAD_FLAG_FIT_BESIDE), part b beside the yielded part a:
// launch_arima_unfinished: *from = the lowest series of a that has fits left (~0u: none).
// launch_arima_pair: one launch fits b beside the fits a has left, a's series a_from ..< a_from + n_a, each part as its
//   own launch would (a as its resume launch, b as launch_arima_fit's fit kernel when b_first, else as its resume launch),
//   about half the warps each.  b's Box-Cox is launch_arima_boxcox.
cudaError_t launch_arima_boxcox(cudaStream_t st, const FitPart &p, const uint64_t *csr_v);
cudaError_t launch_arima_fit(cudaStream_t st, const FitPart &p, const uint64_t *csr_v, const uint32_t *board = nullptr,
                             uint32_t ordinal = 0);
cudaError_t launch_arima_resume(cudaStream_t st, const FitPart &p);
cudaError_t launch_arima_unfinished(cudaStream_t st, const FitPart &a, uint32_t *from);
cudaError_t launch_arima_pair(cudaStream_t st, const FitPart &a, uint32_t a_from, uint32_t n_a, const FitPart &b, bool b_first);
cudaError_t launch_detect_arima(cudaStream_t st, const SeriesEntry *entries, const uint32_t *offsets, const uint32_t *sbase,
                                uint32_t B, uint32_t S, const uint64_t *csr_v, const uint32_t *csr_t, const double *scratch_pred,
                                const double *scratch_lam, const OutCols &out, uint32_t out_cap, uint32_t *stats, int emit_all);

// Oversized buckets (more rows than the shared-memory capacity): global-memory path.
// Sorts the rows of all listed buckets by (hash, key, time), reduces duplicates and writes the
// same per-series arrays / in-place series entries / nsb / npb the group kernel produces.
// `scratch` must hold spill_scratch_bytes(big_rows) bytes.  Returns launches through *launches.
size_t spill_scratch_bytes(uint64_t big_rows);
// Sort a capacity-class bucket list ascending (CUB radix sort over `key_bits` bits); scratch from sort_lists_scratch_bytes(max n).
size_t sort_lists_scratch_bytes(uint32_t max_items);
cudaError_t sort_bucket_list(cudaStream_t st, uint32_t *list, uint32_t n, int key_bits, void *scratch, size_t scratch_bytes);
// CUB exclusive sum of n u32 (temp == nullptr: only sets temp_bytes)
cudaError_t exclusive_scan_u32(void *temp, size_t &temp_bytes, const uint32_t *in, uint32_t *out, int n, cudaStream_t st);
// Optimistic partition (seg.stride != 0): a listed bucket holds min(count, stride) rows in its slot and the rest in
// ovf[0, n_ovf) (every overflow row belongs to a listed bucket).
cudaError_t run_spill(cudaStream_t st, const SegDesc &seg, SeriesEntry *entries, const uint32_t *offsets, const uint32_t *big_list,
                      const uint32_t *big_base, uint32_t n_big, uint64_t big_rows, void *scratch, size_t scratch_bytes,
                      uint64_t *csr_v, uint32_t *csr_t, uint32_t *nsb, uint32_t *npb, int reducer, int *launches,
                      const Row32 *ovf = nullptr, uint32_t n_ovf = 0);

}  // namespace tad

namespace tad {
// Multi-GPU, optimistic partition: pc.p[s] = source rank s's arrival counters (its own for s = me, IPC-mapped otherwise).
// Fills cnt[world x B_local] / total[B_local] for the owned bucket range and adds the sum of this rank's own B_global
// counters (= its rows that passed the filters) to *kept_out.  Two launches.
struct PeerCounters { const uint32_t *p[8]; };
cudaError_t launch_gather_counts(cudaStream_t st, const PeerCounters &pc, int world, uint32_t b_lo, uint32_t B_local, uint32_t slot,
                                 uint32_t *cnt, uint32_t *total, const uint32_t *my_counters, uint32_t B_global, uint32_t *kept_out);
// Multi-GPU: per-source segment offsets and total bucket sizes of this rank's bucket range from the
// all-gathered histograms.  hist_all[r * B_global + b]; range = [b_lo, b_lo + B_local).
cudaError_t launch_segment_scan(cudaStream_t st, const uint32_t *hist_all, uint32_t B_global, uint32_t b_lo, uint32_t B_local,
                                int nseg, uint32_t *seg_off /* nseg x (B_local+1) */, uint32_t *total /* B_local */,
                                unsigned long long *seg_rows /* nseg */,
                                unsigned long long *seg_before = nullptr /* nseg: rows of each source in front of the owned range */);
}
