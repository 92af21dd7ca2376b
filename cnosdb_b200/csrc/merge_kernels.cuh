// merge_kernels.cuh — overlapping chunks of one series: merge on time + last-writer-wins per column, fused with the
// filter / bucket / aggregate of the scan. Replaces, for the aggregate path,
//   DataMerger -> sort_merge -> SortPreservingMergeStream (loser tree)   tskv/src/reader/merge.rs, sort_merge.rs:153-400
//   BatchMergeBuilder::push_row / take_last_and_merge                     tskv/src/reader/batch_builder.rs:74-155
// (and serves memcache rows the same way: the host hands a cache's row group in as one more chunk of raw-encoded pages
// tagged with the cache's file id, reader/iterator.rs:318-343, reader/memcache_reader.rs:33-165).
//
// The reference walks a loser tree row by row. Here nothing is sorted and no merged batch is materialised: the merge
// groups' rows live stream by stream in one row space (OverlapPlan, host_util.h), their timestamps decoded once per page
// set, the queried value columns once per scan (k_decode_warp); then ONE THREAD PER ROW decides by binary search
//   * is this row the first surviving row with its timestamp in (stream, row) order - the "leader" of its merged row?
//   * for every query column: the last surviving row with that timestamp, scanning the streams from the newest file
//     backwards, whose value is non-null - take_last_and_merge's rule; none: the merged value is NULL
// and feeds the merged row to the scan's partial state (closed time ranges, bucket key, count / sum / min / max /
// mean; first / last: only the earliest / latest merged row of the group in a bucket may contribute, and only with a
// non-null value - FirstAccumulator::update_batch on the merged batch, first.rs:139-148).
// A row "survives" when its column group is read by this scan (series selected, not pruned), the pushed row filter
// kept it (DataFilter runs on every chunk BEFORE the merge, reader/iterator.rs:403-413) and no all-fields tombstone
// drops its timestamp.
#pragma once
#include "scan_kernels.cuh"

namespace tskv {

struct MergeParams {
  const int64_t *ts;            // [n_rows] timestamps of the merge rows (decoded once per page set)
  const uint64_t *mcg_row0;     // [n_mcg + 1]
  const uint32_t *mcg_cg;       // [n_mcg] column group of a merge column group
  const uint32_t *mcg_stream;   // [n_mcg]
  const uint32_t *stream_group;      // [n_streams]
  const uint32_t *stream_first_mcg;  // [n_streams + 1]
  const uint32_t *group_first_stream;  // [n_groups + 1]
  const uint8_t *mcg_active;    // [n_mcg] this scan reads the column group (selected series, not pruned)
  const uint64_t *vals;         // [n_cols][n_rows] decoded values of the query columns
  const uint32_t *valid;        // [n_cols][bm_words] validity bitmaps, per merge column group at mcg_bm0
  const uint64_t *mcg_bm0;      // [n_mcg] first bitmap WORD (32 rows) of a merge column group
  const uint32_t *cg_time_page; // column group -> descriptor index of its time page
  const int32_t *cg_slot;       // k_select_cg
  uint64_t n_rows, bm_words;
  uint32_t n_mcg;
  uint32_t sel;                 // the query asks for FIRST / LAST somewhere
};

__device__ __forceinline__ uint64_t merge_lower_bound(const int64_t *ts, uint64_t lo, uint64_t hi, int64_t t) {
  while (lo < hi) {
    const uint64_t mid = lo + ((hi - lo) >> 1);
    if (ts[mid] < t) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}
__device__ __forceinline__ uint64_t merge_upper_bound(const int64_t *ts, uint64_t lo, uint64_t hi, int64_t t) {
  while (lo < hi) {
    const uint64_t mid = lo + ((hi - lo) >> 1);
    if (ts[mid] <= t) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

// merge column group of merge row i
__device__ __forceinline__ uint32_t merge_mcg_of(const MergeParams &M, uint64_t i) {
  uint32_t lo = 0, hi = M.n_mcg;  // last k with mcg_row0[k] <= i
  while (hi - lo > 1) {
    const uint32_t mid = (lo + hi) >> 1;
    if (M.mcg_row0[mid] <= i) lo = mid;
    else hi = mid;
  }
  return lo;
}

// Does merge row i reach the merge? (its column group is read, the row filter kept it; the time-based tombstones are
// the same for every row with this timestamp and are tested once by the caller)
__device__ __forceinline__ bool merge_row_kept(const ScanParams &P, const MergeParams &M, uint64_t i, uint32_t k) {
  if (!M.mcg_active[k]) return false;
  if (!P.row_keep) return true;
  const uint32_t r = (uint32_t)(i - M.mcg_row0[k]);
  const uint32_t *keep = P.row_keep + P.keep_off[M.cg_time_page[M.mcg_cg[k]]];
  return (keep[r >> 5] >> (r & 31)) & 1;
}
// the same when the row's merge column group is not known yet: rows of one stream, k hint = first mcg of the stream
__device__ __forceinline__ bool merge_row_kept_in_stream(const ScanParams &P, const MergeParams &M, uint64_t i, uint32_t s) {
  uint32_t k = M.stream_first_mcg[s];
  const uint32_t k_end = M.stream_first_mcg[s + 1];
  while (k + 1 < k_end && M.mcg_row0[k + 1] <= i) k++;
  return merge_row_kept(P, M, i, k);
}

// (merged_row and merge_value below restate this kernel's leader test, row-level filters and take_last_and_merge rule
// for the column pairs, the medians and the increases: a change to either rule must be made in both.)
// M2: pass 2 of TSKV_AGG_M2 over the merged rows, with the pass-2 column table (k_scan_m2): the same merged rows and cells,
// each M2 column's value adds d = (double)x - (its cell's shift) and d^2 to sum(d) / sum(d^2); other columns are skipped.
template <bool M2>
__global__ void __launch_bounds__(128) k_merge_chunks(const ScanParams P, const MergeParams M) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M.n_rows) return;
  const uint32_t k = merge_mcg_of(M, i);
  if (!merge_row_kept(P, M, i, k)) return;
  const uint32_t s = M.mcg_stream[k], g = M.stream_group[s];
  const uint32_t cg = M.mcg_cg[k];
  const int32_t slot_i = M.cg_slot[cg];
  if (slot_i < 0) return;
  const uint32_t slot = (uint32_t)slot_i;
  const int64_t t = M.ts[i];
  const uint32_t s0 = M.group_first_stream[g], s1 = M.group_first_stream[g + 1];
  const uint32_t series = P.descs[M.cg_time_page[cg]].series_id;

  // ---- leader of the merged row: no surviving row with this timestamp earlier in (stream, row) order
  const uint64_t own0 = M.mcg_row0[M.stream_first_mcg[s]], own1 = M.mcg_row0[M.stream_first_mcg[s + 1]];
  for (uint64_t j = merge_lower_bound(M.ts, own0, i, t); j < i; j++)
    if (merge_row_kept_in_stream(P, M, j, s)) return;
  for (uint32_t s2 = s0; s2 < s; s2++) {
    const uint64_t a = M.mcg_row0[M.stream_first_mcg[s2]], b = M.mcg_row0[M.stream_first_mcg[s2 + 1]];
    for (uint64_t j = merge_lower_bound(M.ts, a, b, t); j < b && M.ts[j] == t; j++)
      if (merge_row_kept_in_stream(P, M, j, s2)) return;
  }
  (void)own1;

  // ---- row-level filters of the merged row: all-fields tombstones, closed time ranges, bucket
  int64_t lim_lo, lim_hi;
  if (!range_span(P, t, lim_lo, lim_hi)) return;
  uint4 tl = make_uint4(0, 0, 0, 0);
  if (P.has_tomb) {
    tl = tomb_lookup(P, series, TSKV_TOMB_ALL);  // .x/.y: the series' row-drop ranges
    int64_t a = INT64_MIN, b = INT64_MAX;
    if (tomb_span(P.tomb_ranges, P.n_tomb_global, t, a, b) | tomb_span(P.tomb_ranges + tl.x, tl.y, t, a, b)) return;
  }
  BucketState bk;
  bk.valid = false; bk.floor_regime = false; bk.lo = 0; bk.hi = 0; bk.idx = 0;
  if (!(P.edges ? locate_bucket<true>(P, t, bk) : locate_bucket<false>(P, t, bk))) {
    report_error(P, TSKV_ERR_BUCKET_RANGE, M.cg_time_page[cg]);
    return;
  }
  // (the edge scans' cell rule: every other scan has cell_buckets = 0, which gives the tumbling one)
  const uint64_t cell = group_cell_base<true>(P, slot) + bucket_cell<true>(P, bk.idx);

  // ---- FIRST / LAST: is this the earliest / latest merged row of the group that lands in this bucket? (the merged rows of
  // a group are one record batch, so its rows of one bucket are one run: a surviving, in-range row of any stream with an
  // earlier / later timestamp inside the bucket takes that place)
  bool is_first = false, is_last = false;
  if (!M2 && M.sel) {
    is_first = is_last = true;
    auto counts = [&](uint64_t j, uint32_t s2) {  // does merge row j reach the aggregate?
      if (!merge_row_kept_in_stream(P, M, j, s2)) return false;
      int64_t x = INT64_MIN, y = INT64_MAX;
      const int64_t tj = M.ts[j];
      if (P.has_tomb && (tomb_span(P.tomb_ranges, P.n_tomb_global, tj, x, y) | tomb_span(P.tomb_ranges + tl.x, tl.y, tj, x, y))) return false;
      return range_span(P, tj, x, y);
    };
    for (uint32_t s2 = s0; s2 < s1 && (is_first || is_last); s2++) {
      const uint64_t a = M.mcg_row0[M.stream_first_mcg[s2]], b = M.mcg_row0[M.stream_first_mcg[s2 + 1]];
      const uint64_t lb = merge_lower_bound(M.ts, a, b, t), ub = merge_upper_bound(M.ts, lb, b, t);
      for (uint64_t j = lb; is_first && j > a && M.ts[j - 1] >= bk.lo; j--)
        if (counts(j - 1, s2)) is_first = false;
      for (uint64_t j = ub; is_last && j < b && M.ts[j] <= bk.hi; j++)
        if (counts(j, s2)) is_last = false;
    }
  }

  // ---- per query column: the last surviving non-null value with this timestamp (take_last_and_merge)
  for (uint32_t c = 0; c < P.n_cols; c++) {
    const ColState cs = P.cols[c];
    if (M2 && !(cs.agg_mask & TSKV_AGG_M2)) continue;
    bool have = false;
    uint64_t v = 0;
    bool masked = false;  // (series, column) tombstone: the column reads as NULL at this timestamp in every chunk
    if (P.has_tomb) {
      const uint4 tc = tomb_lookup(P, series, cs.column_id);
      int64_t x = INT64_MIN, y = INT64_MAX;
      masked = tomb_span(P.tomb_ranges + tc.z, tc.w, t, x, y);
    }
    for (uint32_t s2 = s1; !masked && !have && s2-- > s0;) {
      const uint64_t a = M.mcg_row0[M.stream_first_mcg[s2]], b = M.mcg_row0[M.stream_first_mcg[s2 + 1]];
      const uint64_t lb = merge_lower_bound(M.ts, a, b, t);
      uint64_t ub = lb;
      while (ub < b && M.ts[ub] == t) ub++;
      uint32_t k2 = M.stream_first_mcg[s2 + 1];  // merge column group of row j, walking backwards
      for (uint64_t j = ub; !have && j-- > lb;) {
        while (M.mcg_row0[k2] > j) k2--;  // (k2 starts one past the stream's last merge column group)
        if (!merge_row_kept(P, M, j, k2)) continue;
        const uint32_t r = (uint32_t)(j - M.mcg_row0[k2]);
        const uint32_t w = M.valid[(uint64_t)c * M.bm_words + M.mcg_bm0[k2] + (r >> 5)];
        if ((w >> (r & 31)) & 1) {
          have = true;
          v = M.vals[(uint64_t)c * M.n_rows + j];
        }
      }
    }
    if (M2 && have) {
      const uint8_t pt = cs.phys_type;
      const double x = pt == TSKV_PT_F64 ? __longlong_as_double((long long)v) : pt == TSKV_PT_I64 ? (double)(int64_t)v : (double)v;
      const double d = x - __longlong_as_double((long long)P.state[cs.count_off + cell]);
      atomicAdd(reinterpret_cast<double *>(P.state + cs.sum_off + cell), d);
      atomicAdd(reinterpret_cast<double *>(P.state + cs.sumhi_off + cell), d * d);
    } else if (have) {
      const uint8_t pt = cs.phys_type, mask = cs.agg_mask;
      const int64_t key = okey(v, pt);
      atomicAdd(reinterpret_cast<unsigned long long *>(P.state + cs.count_off + cell), 1ull);
      if (mask & (TSKV_AGG_SUM | TSKV_AGG_MEAN)) {
        if (pt == TSKV_PT_F64) atomicAdd(reinterpret_cast<double *>(P.state + cs.sum_off + cell), __longlong_as_double((long long)v));
        else add_int_sum(P.state + cs.sum_off + cell, P.state + cs.sumhi_off + cell, mask, v, pt == TSKV_PT_I64 ? ((int64_t)v >> 63) : 0);
      }
      if (mask & TSKV_AGG_MIN) atomicMin(reinterpret_cast<long long *>(P.state + cs.min_off + cell), (long long)key);
      if (mask & TSKV_AGG_MAX) atomicMax(reinterpret_cast<long long *>(P.state + cs.max_off + cell), (long long)key);
      if (M.sel && (mask & (TSKV_AGG_FIRST | TSKV_AGG_LAST))) {
        int64_t kf = t, kl = t;
        if (P.slot_bits) {
          const uint64_t base = P.edges ? key_base<true>(P, (int64_t)bk.idx) : key_base<false>(P, (int64_t)bk.idx);
          kf = (int64_t)((((uint64_t)t - base) << P.slot_bits) | slot);
          kl = (int64_t)((((uint64_t)t - base) << P.slot_bits) | (P.slot_max - slot));
        }
        if ((mask & TSKV_AGG_FIRST) && is_first) atomic_select_pair<true>(P.state + cs.first_off + 2 * cell, kf, v);
        if ((mask & TSKV_AGG_LAST) && is_last) atomic_select_pair<false>(P.state + cs.last_off + 2 * cell, kl, v);
      }
    }
  }
}

// The column pairs over the merged rows (pass 1 / pass 2 of k_scan_pair): one thread per merge row; the leader of a merged
// row that survives the row-level filters takes, for each pair, the merged x and y values as k_merge_chunks takes them
// for its columns (column tombstones, then the newest surviving non-null value with this timestamp) and adds the pair
// when both exist. The leader test, the row-level filters (merged_row) and the take_last_and_merge rule (merge_value)
// restate k_merge_chunks' so that the existing kernel's code stays as it is: a change to either must be made in both.
__device__ __forceinline__ bool merge_value(const ScanParams &P, const MergeParams &M, uint32_t c, uint32_t series, int64_t t,
                                            uint32_t s0, uint32_t s1, uint64_t &v) {
  if (P.has_tomb) {
    const uint4 tc = tomb_lookup(P, series, P.cols[c].column_id);
    int64_t x = INT64_MIN, y = INT64_MAX;
    if (tomb_span(P.tomb_ranges + tc.z, tc.w, t, x, y)) return false;
  }
  for (uint32_t s2 = s1; s2-- > s0;) {
    const uint64_t a = M.mcg_row0[M.stream_first_mcg[s2]], b = M.mcg_row0[M.stream_first_mcg[s2 + 1]];
    const uint64_t lb = merge_lower_bound(M.ts, a, b, t);
    uint64_t ub = lb;
    while (ub < b && M.ts[ub] == t) ub++;
    uint32_t k2 = M.stream_first_mcg[s2 + 1];
    for (uint64_t j = ub; j-- > lb;) {
      while (M.mcg_row0[k2] > j) k2--;
      if (!merge_row_kept(P, M, j, k2)) continue;
      const uint32_t r = (uint32_t)(j - M.mcg_row0[k2]);
      if ((M.valid[(uint64_t)c * M.bm_words + M.mcg_bm0[k2] + (r >> 5)] >> (r & 31)) & 1) {
        v = M.vals[(uint64_t)c * M.n_rows + j];
        return true;
      }
    }
  }
  return false;
}

// A merged row of the column pairs and the medians: the leader of its timestamp and group, as k_merge_chunks leads one
// (merge row i is kept and no earlier kept row of its stream, and no kept row of an older stream, has its timestamp),
// past the row-level filters (time ranges, row-drop tombstones, its bucket). Sets the row's cell, timestamp and series
// and its group's streams [s0, s1) (merge_value's arguments).
struct MergedRow {
  uint64_t cell;
  int64_t t;
  uint32_t series, s0, s1;
};
__device__ __forceinline__ bool merged_row(const ScanParams &P, const MergeParams &M, uint64_t i, MergedRow &mr) {
  const uint32_t k = merge_mcg_of(M, i);
  if (!merge_row_kept(P, M, i, k)) return false;
  const uint32_t s = M.mcg_stream[k], g = M.stream_group[s];
  const uint32_t cg = M.mcg_cg[k];
  const int32_t slot_i = M.cg_slot[cg];
  if (slot_i < 0) return false;
  const int64_t t = M.ts[i];
  const uint32_t s0 = M.group_first_stream[g], s1 = M.group_first_stream[g + 1];
  const uint32_t series = P.descs[M.cg_time_page[cg]].series_id;
  const uint64_t own0 = M.mcg_row0[M.stream_first_mcg[s]];
  for (uint64_t j = merge_lower_bound(M.ts, own0, i, t); j < i; j++)
    if (merge_row_kept_in_stream(P, M, j, s)) return false;
  for (uint32_t s2 = s0; s2 < s; s2++) {
    const uint64_t a = M.mcg_row0[M.stream_first_mcg[s2]], b = M.mcg_row0[M.stream_first_mcg[s2 + 1]];
    for (uint64_t j = merge_lower_bound(M.ts, a, b, t); j < b && M.ts[j] == t; j++)
      if (merge_row_kept_in_stream(P, M, j, s2)) return false;
  }
  int64_t lo, hi;
  if (!range_span(P, t, lo, hi)) return false;
  if (P.has_tomb) {
    const uint4 tl = tomb_lookup(P, series, TSKV_TOMB_ALL);
    if (tomb_span(P.tomb_ranges, P.n_tomb_global, t, lo, hi) | tomb_span(P.tomb_ranges + tl.x, tl.y, t, lo, hi)) return false;
  }
  BucketState bk;
  bk.valid = false; bk.floor_regime = false; bk.lo = 0; bk.hi = 0; bk.idx = 0;
  if (!(P.edges ? locate_bucket<true>(P, t, bk) : locate_bucket<false>(P, t, bk))) return false;  // (k_merge_chunks reports it)
  mr.cell = group_cell_base<true>(P, (uint32_t)slot_i) + bucket_cell<true>(P, bk.idx);
  mr.t = t;
  mr.series = series;
  mr.s0 = s0;
  mr.s1 = s1;
  return true;
}

template <bool PASS2>
__global__ void __launch_bounds__(128) k_merge_pairs_rows(const ScanParams P, const MergeParams M, const PairCol *pairs, uint32_t n_pairs) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  MergedRow mr;
  if (i >= M.n_rows || !merged_row(P, M, i, mr)) return;
  for (uint32_t p = 0; p < n_pairs; p++) {
    const PairCol pc = pairs[p];
    uint64_t xv, yv;
    if (!merge_value(P, M, pc.qx, mr.series, mr.t, mr.s0, mr.s1, xv) || !merge_value(P, M, pc.qy, mr.series, mr.t, mr.s0, mr.s1, yv))
      continue;
    PairAcc acc;
    pair_start<PASS2>(P, pc, mr.cell, acc);
    pair_add<PASS2>(acc, pair_f64(xv, pc.x_pt), pair_f64(yv, pc.y_pt));
    pair_flush<PASS2>(P, pc, mr.cell, acc);
  }
}

// One selection pass of the medians over the merged rows (k_scan_median's pass): one thread per merge row; the leader of
// a merged row adds, for each median, the operand's merged value (merge_value) to its cell.
__global__ void __launch_bounds__(128) k_merge_median_rows(const ScanParams P, const MergeParams M, const MedianCol *meds, uint32_t n_meds,
                                                           const MedianArgs A) {
  if (*(volatile unsigned long long *)A.unresolved == 0) return;
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  MergedRow mr;
  if (i >= M.n_rows || !merged_row(P, M, i, mr)) return;
  for (uint32_t m = 0; m < n_meds; m++) {
    const MedianCol mc = meds[m];
    uint64_t v;
    if (!merge_value(P, M, mc.qcol, mr.series, mr.t, mr.s0, mr.s1, v)) continue;
    MedianRun run;
    median_open(mc, A, P.n_cells, mr.cell, run);
    median_add(mc, A, P.n_cells, run, median_ukey(v, mc.phys_type));
    median_flush(mc, A, P.n_cells, run);
  }
}

// The increases over the merged rows (k_scan_increase's pages): one thread per (merge row, increase = blockIdx.y); the
// leader of a merged row that survives the row-level filters (merged_row) and holds a merged value of the operand
// (merge_value) writes record rec0 + i, one point: k_increase_stitch pairs it with the point before it in its series,
// as it pairs the pages' boundary points, so a large merge group runs one thread per row, not one per group.
__global__ void __launch_bounds__(128) k_merge_increase(const ScanParams P, const MergeParams M, const IncreaseCol *incs, const IncreaseArgs A,
                                                        uint32_t rec0) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  MergedRow mr;
  if (i >= M.n_rows || !merged_row(P, M, i, mr)) return;
  const IncreaseCol ic = incs[blockIdx.y];
  uint64_t v;
  if (!merge_value(P, M, ic.qcol, mr.series, mr.t, mr.s0, mr.s1, v)) return;
  IncreaseRun run;
  increase_begin(run);
  increase_add(P.state, ic, run, mr.cell, mr.t, v);
  increase_end(P.state, ic, A, blockIdx.y, rec0 + i, (uint32_t)M.cg_slot[M.mcg_cg[merge_mcg_of(M, i)]], run);
}

}  // namespace tskv
