// scan_kernels.cuh — sm_90a kernels of the tskv scan path:
//   k_select_cg / k_flag_items / k_scan_blocks / k_scatter_items : series selection -> compacted,
//       kind-sorted work list (replaces get_series_id_by_filter's consumer side,
//       tskv/src/reader/iterator.rs:915-929 + SeriesGroupBatchReaderFactory::create :123-264)
//   k_scan_aggregate<TK,VK> : fused decode -> closed time-range filter -> bucket id -> reduce
//       (replaces ColumnGroupReader::read + decode_pages + DataFilter + the DataFusion
//        projection/AggregateExec above the scan; SURVEY.md §3.1 hot loops A, B and C)
//   k_export_pairs / k_mask_values / k_finalize : partial state -> dense Arrow-style result
//   (decode-only, Page::to_arrow_array: decode_kernels.cuh)
#pragma once
#include <type_traits>

#include "cursors.cuh"

namespace tskv {

constexpr uint32_t FULL = 0xffffffffu;
constexpr int MAX_RANGES = 8;
constexpr int N_TK = 3;  // time-cursor specialisations: RLE, S8B scaled, generic
constexpr int N_VK = 3;  // value-cursor specialisations: S8B zig-zag, gorilla, generic
constexpr int N_SERIAL_BINS = N_TK * N_VK;  // bins 0-8: time class * N_VK + value class
// + the short-page bins: zig-zag simple8b or gorilla values of at most SHORT_PAGE_ROWS rows with RLE / simple8b
// timestamps. The kernel of the matching class (serial_bin_of) runs them; they stay apart because plan_bin_parts sizes
// a bin's parts from its longest page (short pages in a bin with long ones would get coarser parts), because each
// bin stream's priority is its chunk_cost rank among all the bins, and because the dominant_kernel_bin counter and
// the benchmark report these bin numbers.
constexpr uint32_t SHORT_PAGE_ROWS = 1024;
enum { BIN_SHORT_RLE_S8B = N_SERIAL_BINS, BIN_SHORT_S8B_S8B = N_SERIAL_BINS + 1, BIN_SHORT_RLE_GOR = N_SERIAL_BINS + 2,
       BIN_SHORT_S8B_GOR = N_SERIAL_BINS + 3 };
constexpr int N_BINS = N_SERIAL_BINS + 4;

enum { TK_RLE = 0, TK_S8B = 1, TK_GEN = 2 };
enum { VK_S8B = 0, VK_GOR = 1, VK_GEN = 2 };

__host__ __device__ inline int time_class(uint8_t dk) {
  return dk == DK_RLE_SC ? TK_RLE : dk == DK_S8B_SC ? TK_S8B : TK_GEN;
}
__host__ __device__ inline int value_class(uint8_t dk) {
  return dk == DK_S8B_ZZ ? VK_S8B : dk == DK_GORILLA ? VK_GOR : VK_GEN;
}

// Per query column: where its partial state lives (offsets in 8-byte units into `state`).
struct ColState {
  uint64_t count_off;  // u64 count[n_cells]                       (always)
  uint64_t sum_off;    // i64 wrapping / f64 sum[n_cells]           (SUM | MEAN)
  uint64_t min_off;    // ordered i64 key[n_cells]                  (MIN)
  uint64_t max_off;    // ordered i64 key[n_cells]                  (MAX)
  uint64_t first_off;  // {i64 key, u64 val}[n_cells], 16B aligned  (FIRST)
  uint64_t last_off;   // {i64 key, u64 val}[n_cells], 16B aligned  (LAST)
  uint64_t sumhi_off;  // i64 high word of the exact 128-bit integer sum (MEAN on i64/u64 columns)
  // word offsets of the same arrays inside the per-CTA shared-memory table (GROUP BY bucket only)
  uint32_t s_count, s_sum, s_hi, s_min, s_max, s_pad;
  uint16_t column_id;
  uint8_t phys_type;
  uint8_t agg_mask;
  uint32_t pad;
};

constexpr int SCAN_THREADS = 128;  // threads per CTA of the fused scan kernels

struct ScanParams {
  const uint8_t *arena;
  const tskv_page_desc *descs;   // device copy; .reserved = DK_* kind
  const uint32_t *time_page_of;  // field page -> its column group's time page
  // compacted work list (kind-sorted)
  const uint32_t *work_page;
  const uint32_t *work_slot;
  const uint8_t *work_qcol;
  const uint32_t *bin_cstart;  // [N_BINS + 1] starts of the kind bins in the work list
  const ColState *cols;
  uint64_t *state;
  uint32_t *task_counter;       // [N_BINS] dynamic chunk schedulers
  int32_t *status;              // first error (0 = ok)
  unsigned long long *err_page; // page of the first error
  unsigned long long *stats;    // [0] points decoded, [1] rows in range
  tskv_time_range ranges[MAX_RANGES];
  uint32_t n_ranges;
  int64_t width;         // <= 0: single bucket
  int64_t origin_mod;    // origin % width; a sliding scan's panes: origin % window, which may lie outside (-width, width)
  // Rows whose dividend t - origin_mod + width does not wrap: [wrap_lo, floor_cap] (set by the host; a tumbling scan has
  // wrap_lo = INT64_MIN). Floor-regime buckets end at floor_cap; rows below wrap_lo are located one by one.
  int64_t floor_cap, wrap_lo;
  int64_t first_bucket_start;
  uint32_t n_buckets;
  uint32_t group_by_series;
  uint64_t n_cells;
  // GROUP BY tags: group of every slot, < n_groups with n_groups * n_buckets < 2^32 (host-checked); null otherwise
  const uint32_t *slot_group;
  // first/last tie-break key. slot_bits == 0 (one slot per cell): key = timestamp itself.
  // Otherwise key = rel << slot_bits | slot with rel = t - (bucket_start - width) in (0, 2*width)
  // for bucketed scans and rel = t - rel_base for unbucketed ones; the host checked the bit budget.
  uint32_t slot_bits;
  uint32_t slot_max;     // (1 << slot_bits) - 1
  int64_t rel_base;
  // Per-CTA partial table in shared memory (count/sum/min/max of every (column, bucket) cell): all warps
  // of the grid work on the same bucket at the same time, so flushing straight to global memory
  // serialises every warp on a handful of L2 atomics. Used when GROUP BY bucket and the table fits.
  uint32_t use_smem;
  uint32_t smem_words;   // table size in 8-byte words
  uint32_t n_cols;
  // TsmTombstone ranges of the page set (tskvgpu_pages_set_tombstones): ranges [0, n_tomb_global) drop rows of every
  // series; sorted keys (series << 32 | column, column = TSKV_TOMB_ALL: drop rows of the series, else: the
  // column reads as NULL) index the rest through the CSR offsets.
  uint32_t has_tomb;
  const uint64_t *tomb_keys;
  const uint32_t *tomb_off;
  const tskv_time_range *tomb_ranges;
  uint32_t n_tomb_keys;
  uint32_t n_tomb_global;
  // Row filter (tskv_field_predicate): one keep bit per row of every column group, written by k_row_filter before the
  // fused kernels; words of a group start at row_keep + keep_off[index of the group's time page]. null: no predicates.
  const uint32_t *row_keep;
  const uint32_t *keep_off;
  // Restart points of the page set (cursors.cuh, SkipEntry; null: none). skip_off[page] = index of the page's first
  // entry in `skip` (entry j - 1 = the state at row j * SKIP_ROWS) or SKIP_NONE. A bin whose pages are cut into
  // bin_parts[bin] > 1 parts of bin_part_rows[bin] rows (a multiple of SKIP_ROWS) runs parts x as many chunks; all
  // lanes of a chunk decode the SAME part of 32 different pages.
  const uint32_t *skip_off;
  const SkipEntry *skip;
  uint32_t bin_parts[N_BINS];
  uint32_t bin_part_rows[N_BINS];
  // page_narrow[page] = 1: every value of the simple8b integer page lies in [-2^31, 2^31) (i64) or [0, 2^31) (u64)
  // (k_build_skip, from the decoded values; null or 0: not known). Chunks whose pages are all narrow accumulate in 32-bit
  // arithmetic.
  const uint8_t *page_narrow;
};

// First cell of the group a work item's series belongs to: GROUP BY tags slot_group[slot], GROUP BY series the slot
// itself, GROUP BY bucket the one group. Read once per page.
__device__ __forceinline__ uint64_t group_cell_base(const ScanParams &P, uint32_t slot) {
  if (P.slot_group) return (uint64_t)__ldg(P.slot_group + slot) * P.n_buckets;
  return P.group_by_series ? (uint64_t)slot * P.n_buckets : 0;
}

// ------------------------------------------------------------------------------------------------
// selection / compaction
// ------------------------------------------------------------------------------------------------
// Series selection -> slot of every column group, in two steps: one thread per SELECTED id finds the id's rank among
// the page set's series (binary search in the sorted distinct ids) and writes its position in the selection list to
// rank_slot[rank] (memset to -1 before); then one thread per column group gathers rank_slot[rank of its series].
// (Round 1 searched the selection list once per column group: 10 x the dependent loads for a 10 % selection.)
__global__ void k_select_ids(const uint32_t *set_series, uint32_t n_set_series, const uint32_t *series_ids, uint32_t n_series,
                             int32_t *rank_slot) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_series) return;
  const uint32_t id = __ldg(series_ids + i);
  uint32_t lo = 0, hi = n_set_series;
  while (lo < hi) {
    const uint32_t mid = (lo + hi) >> 1;
    if (__ldg(set_series + mid) < id) lo = mid + 1; else hi = mid;
  }
  if (lo < n_set_series && __ldg(set_series + lo) == id) rank_slot[lo] = (int32_t)i;
}
__global__ void k_select_cg(uint32_t n_cg, const int32_t *rank_slot, const uint32_t *cg_series_rank, int32_t *cg_slot) {
  const uint32_t cg = blockIdx.x * blockDim.x + threadIdx.x;
  if (cg >= n_cg) return;
  const uint32_t rank = cg_series_rank[cg];
  cg_slot[cg] = rank_slot ? rank_slot[rank] : (int32_t)rank;  // no selection list: every series, slot = rank
}

// The pushed field predicates of a query (row filter: k_row_filter; value-statistics pruning: below).
struct PredicateSet {
  tskv_field_predicate p[TSKV_MAX_PREDICATES];
  uint32_t n;
  uint32_t pad;
};

// ---- value-statistics pruning (filter_column_groups with PageMeta.statistics, tskv/src/reader/chunk.rs:12-50 +
// reader/column_group/statistics.rs:11-80: PruningPredicate over the pages' min / max) ------------------------------
// Per field page: {min key, max key} of its non-null (f64: non-NaN) values as ordered i64 keys (okey; -0.0 counted as
// +0.0 so that key order = numeric order). No such value: {INT64_MAX, INT64_MIN}. A page that did not decode:
// {INT64_MIN, INT64_MAX} = nothing can be ruled out (the scan reports its error). Built once per page set, on the first
// scan that carries field predicates (k_page_stats); the reference keeps the same numbers in PageMeta.statistics.
__host__ __device__ inline int64_t stats_key(uint64_t v, uint8_t pt) {
  if (pt == TSKV_PT_F64 && v == 0x8000000000000000ull) v = 0;  // -0.0 == +0.0
  uint64_t flip = pt == TSKV_PT_U64 ? 0x8000000000000000ull
                  : pt == TSKV_PT_F64 ? (uint64_t)(((int64_t)v >> 63) & 0x7fffffffffffffffll)
                                      : 0ull;
  return (int64_t)(v ^ flip);
}
// Can NO value in [kmin, kmax] satisfy `value <op> constant`? (what PruningPredicate derives from min / max)
__host__ __device__ inline bool stats_rule_out(uint8_t pt, uint8_t op, uint64_t constant, int64_t kmin, int64_t kmax) {
  if (pt == TSKV_PT_F64) {
    const uint64_t a = constant & 0x7fffffffffffffffull;
    if (a > 0x7ff0000000000000ull) return true;  // NaN constant: the comparison is never TRUE
  }
  if (kmin > kmax) return true;                  // no value at all: every row is NULL, never TRUE
  const int64_t kc = stats_key(constant, pt);
  switch (op) {
    case TSKV_CMP_EQ: return kc < kmin || kc > kmax;
    case TSKV_CMP_NE: return kmin == kmax && kmin == kc;
    case TSKV_CMP_LT: return kmin >= kc;
    case TSKV_CMP_LE: return kmin > kc;
    case TSKV_CMP_GT: return kmax <= kc;
    case TSKV_CMP_GE: return kmax < kc;
    default: return false;
  }
}
// Is the column group whose pages are descriptors (tp, end) ruled out by some predicate's page statistics?
// (a predicate column the group does not hold is not ruled out here: the row filter drops its rows)
__device__ __forceinline__ bool cg_ruled_out_by_stats(const tskv_page_desc *descs, uint64_t tp, uint64_t end, const PredicateSet &preds,
                                                      const int64_t *page_stats) {
  for (uint32_t k = 0; k < preds.n; k++) {
    const tskv_field_predicate fp = preds.p[k];
    for (uint64_t p = tp + 1; p < end; p++)
      if (descs[p].column_id == fp.column_id) {
        if (descs[p].phys_type == fp.phys_type && stats_rule_out(fp.phys_type, fp.op, fp.value, page_stats[2 * p], page_stats[2 * p + 1])) return true;
        break;
      }
  }
  return false;
}

__device__ __forceinline__ int find_qcol(const ColState *cols, uint32_t n_cols, uint16_t column_id) {
  for (uint32_t c = 0; c < n_cols; c++)
    if (cols[c].column_id == column_id) return (int)c;
  return -1;
}

// One thread per item (field page, in kind-sorted order): selected? -> flag (query column + 1, bit 7 =
// "this item also brings its column group's time page"), per-block counts and the byte/page counters
// of the reference's reader metrics (column_group/mod.rs:141-193), split per decode-kind bin.
// counters: [0] pages, [1] bytes, [2 + bin] bytes read by bin's fused kernel.
// Statistics pruning (filter_column_groups, tskv/src/reader/chunk.rs:12-50 with the column group's time_range(),
// tsm/column_group.rs:9-17): a group whose [min_ts, max_ts] overlaps none of the query's time ranges is dropped here,
// so its pages are neither gathered nor decoded. counters[2 + N_BINS] counts the pruned groups' field pages.
struct PruneRanges {
  tskv_time_range r[MAX_RANGES];
  uint32_t n;
  uint32_t pad;
};
// item_info[i] = {page, column group, page size, column id | phys type << 16 | decode kind << 24} (built at upload: one
// coalesced 16-byte load per item instead of the item -> page -> descriptor chain).
__global__ void k_flag_items(const tskv_page_desc *descs, const uint4 *item_info,
                             const uint32_t *cg_time_page, uint32_t n_items,
                             const int32_t *cg_slot, const ColState *cols, uint32_t n_cols,
                             const uint32_t *bin_start, uint8_t *item_flag, uint32_t *block_count,
                             unsigned long long *counters, int32_t *status, const tskv_time_range *cg_bounds,
                             const PruneRanges prune, const uint8_t *cg_merge, const int64_t *page_stats,
                             const PredicateSet preds, uint64_t n_descs, uint32_t n_cg) {
  __shared__ uint32_t s_cnt;
  __shared__ unsigned long long s_pages, s_bytes[N_BINS];
  if (threadIdx.x == 0) { s_cnt = 0; s_pages = 0; }
  if (threadIdx.x < N_BINS) s_bytes[threadIdx.x] = 0;
  __syncthreads();
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  bool sel = false;
  if (i < n_items) {
    const uint4 info = __ldg(item_info + i);
    const uint32_t p = info.x, cg = info.y;
    struct { uint32_t size; uint16_t column_id; uint8_t phys_type, reserved; } d = {info.z, (uint16_t)(info.w & 0xffff), (uint8_t)((info.w >> 16) & 0xff), (uint8_t)(info.w >> 24)};
    int qc = find_qcol(cols, n_cols, d.column_id);
    bool first_sel = false;
    bool in_time = true;
    if (cg_bounds && prune.n) {  // TimeRange::overlaps against the group's statistics
      const tskv_time_range b = cg_bounds[cg];
      in_time = false;
      for (uint32_t k = 0; k < prune.n; k++) in_time = in_time || (b.min_ts <= prune.r[k].max_ts && b.max_ts >= prune.r[k].min_ts);
    }
    if (in_time && page_stats && qc >= 0 && cg_slot[cg] >= 0) {  // value statistics against the pushed predicates
      const uint32_t tp0 = cg_time_page[cg];
      const uint64_t end = cg + 1 < n_cg ? (uint64_t)cg_time_page[cg + 1] : n_descs;
      if (cg_ruled_out_by_stats(descs, tp0, end, preds, page_stats)) in_time = false;
    }
    if (!in_time && qc >= 0 && cg_slot[cg] >= 0 && !(cg_merge && cg_merge[cg])) atomicAdd(&counters[2 + N_BINS], 1ull);
    // (column groups of overlapping chunks go through the merge pass instead, merge_kernels.cuh)
    if (qc >= 0 && cg_slot[cg] >= 0 && in_time && !(cg_merge && cg_merge[cg])) {
      if (cols[qc].phys_type != d.phys_type) {
        atomicCAS(status, 0, TSKV_ERR_INVALID_ARG);
      } else {
        sel = true;
        unsigned long long bytes = d.size, pages = 1;
        // The time page of a column group is brought along (PCIe gather, CRC check, byte counters) by the first selected
        // field page of the group IN EACH DECODE-KIND BIN: the bins' gathers and fused kernels run on different streams,
        // so a bin must not rely on another bin having copied the time page (a series with an i64 and an f64 field
        // selected together lands in two bins). Field pages of a group are contiguous after the time page and share its
        // time class, so "same bin" is "same value class".
        // The reader metrics (page_read_count / page_read_bytes) count the time page once per column group.
        uint32_t tp = cg_time_page[cg];
        first_sel = true;
        bool first_in_group = true;
        const int vclass = value_class(d.reserved);
        for (uint32_t q = tp + 1; q < p; q++)
          if (find_qcol(cols, n_cols, descs[q].column_id) >= 0) {
            first_in_group = false;
            if (value_class(descs[q].reserved) == vclass) { first_sel = false; break; }
          }
        if (first_in_group) { bytes += descs[tp].size; pages += 1; }
        int bin = 0;
        for (int k = 1; k < N_BINS; k++) bin += (i >= bin_start[k]) ? 1 : 0;
        atomicAdd(&s_bytes[bin], bytes);
        atomicAdd(&s_pages, pages);
      }
    }
    item_flag[i] = sel ? (uint8_t)((qc + 1) | (first_sel ? 0x80 : 0)) : 0;
  }
  uint32_t m = __ballot_sync(FULL, sel);
  if ((threadIdx.x & 31) == 0 && m) atomicAdd(&s_cnt, __popc(m));
  __syncthreads();
  if (threadIdx.x == 0) {
    block_count[blockIdx.x] = s_cnt;
    if (s_pages) atomicAdd(&counters[0], s_pages);
  }
  if (threadIdx.x < N_BINS && s_bytes[threadIdx.x]) {
    atomicAdd(&counters[1], s_bytes[threadIdx.x]);
    atomicAdd(&counters[2 + threadIdx.x], s_bytes[threadIdx.x]);
  }
}

// ------------------------------------------------------------------------------------------------
// Work list driven by the SELECTION (round 2): one thread per selected series walks that series' column groups and
// their field pages, so the cost follows the selection (C4: 10 % of the series) instead of the page set. Two passes
// over the same walk - count per (decode-kind bin, query column) bucket, then place - with a block-local histogram in
// shared memory so that the global atomics are one per (block, bucket). Inside a bucket the order is arbitrary (the
// fused kernels only need warps that are homogeneous in codec and, for GROUP BY bucket, in column). A (bin, column)
// bucket is split in two by the page's narrow flag (WL_SUB buckets, ScanParams.page_narrow): its wide pages come first,
// then its narrow ones, so that all chunks of the bucket but the one across the boundary are uniformly narrow or wide.
// Same outputs as k_flag_items / k_scan_blocks / k_scatter_items: work_page / work_slot / work_qcol (bit 7 = "brings
// the column group's time page": the first selected field page of each value class of a group), bin_cstart, the
// reader counters, statistics pruning.
// ------------------------------------------------------------------------------------------------
constexpr int WL_THREADS = 256;
constexpr uint32_t WL_SUB = 2;  // work-list buckets per (bin, query column): wide pages, narrow pages
struct WorkListArgs {
  const tskv_page_desc *descs;
  uint64_t n_descs;
  const uint32_t *cg_time_page;  // [n_cg]
  uint32_t n_cg;
  const uint32_t *rank_cg_start; // [n_set_series + 1] CSR: column groups of the series with this rank
  const uint32_t *rank_cg;
  const uint8_t *page_bin;       // [n_descs] decode-kind bin of a field page
  const uint8_t *page_narrow;    // [n_descs] narrow flags (null: every page is wide)
  const uint32_t *set_series;    // the page set's distinct series ids, ascending
  uint32_t n_set_series;
  const uint32_t *series_ids;    // the selection (null: every series, slot = rank)
  uint32_t n_sel;                // threads: selected ids, or n_set_series
  // GROUP BY tags: thread i walks slot walk[i], the slots stably sorted by group, so that the items of a (bin, column)
  // bucket come group by group and a warp's 32 pages mostly share a group (null: thread i walks slot i)
  const uint32_t *walk;
  const ColState *cols;
  uint32_t n_cols;
  const tskv_time_range *cg_bounds;  // statistics pruning (null: none)
  PruneRanges prune;
  const uint8_t *cg_merge;       // column groups of overlapping chunks go through the merge pass
  const int64_t *page_stats;     // value-statistics pruning against `preds` (null: none)
  PredicateSet preds;
  uint32_t *bucket_count;        // [N_BINS * n_cols * WL_SUB] totals (pass 1), then running cursors (pass 2)
  uint32_t *bucket_off;          // [N_BINS * n_cols * WL_SUB + 1] exclusive offsets (k_worklist_offsets)
  uint32_t *work_page, *work_slot;
  uint8_t *work_qcol;
  unsigned long long *counters;  // [0] pages [1] bytes [2 + bin] bytes per bin [2 + N_BINS] pruned pages
  int32_t *status;
};

// Work-list bucket of a page: (bin, query column, narrow flag).
__device__ __forceinline__ uint32_t worklist_key(const WorkListArgs &A, uint32_t page, uint32_t bin, uint32_t qc) {
  return (bin * A.n_cols + qc) * WL_SUB + ((A.page_narrow && A.page_narrow[page]) ? 1u : 0u);
}

// Walks the items of selected series i; F(page, bin, qcol, with_time, desc).
template <typename F>
__device__ __forceinline__ void worklist_walk(const WorkListArgs &A, uint32_t i, bool count_stats, F &&emit) {
  uint32_t rank = i;
  if (A.series_ids) {
    const uint32_t id = __ldg(A.series_ids + i);
    uint32_t lo = 0, hi = A.n_set_series;
    while (lo < hi) {
      const uint32_t mid = (lo + hi) >> 1;
      if (__ldg(A.set_series + mid) < id) lo = mid + 1; else hi = mid;
    }
    if (lo >= A.n_set_series || __ldg(A.set_series + lo) != id) return;  // a selected id this page set does not hold
    rank = lo;
  }
  const uint32_t c0 = __ldg(A.rank_cg_start + rank), c1 = __ldg(A.rank_cg_start + rank + 1);
  for (uint32_t k = c0; k < c1; k++) {
    const uint32_t cg = __ldg(A.rank_cg + k);
    if (A.cg_merge && A.cg_merge[cg]) continue;
    bool in_time = true;
    if (A.cg_bounds && A.prune.n) {  // TimeRange::overlaps against the group's statistics
      const tskv_time_range b = A.cg_bounds[cg];
      in_time = false;
      for (uint32_t r = 0; r < A.prune.n; r++) in_time = in_time || (b.min_ts <= A.prune.r[r].max_ts && b.max_ts >= A.prune.r[r].min_ts);
    }
    const uint32_t tp = __ldg(A.cg_time_page + cg);
    const uint64_t end = cg + 1 < A.n_cg ? (uint64_t)__ldg(A.cg_time_page + cg + 1) : A.n_descs;
    if (in_time && A.page_stats && cg_ruled_out_by_stats(A.descs, tp, end, A.preds, A.page_stats)) in_time = false;
    uint32_t seen_classes = 0;  // value classes that already brought the time page
    bool any = false;
    for (uint64_t p = (uint64_t)tp + 1; p < end; p++) {
      const tskv_page_desc d = A.descs[p];
      const int qc = find_qcol(A.cols, A.n_cols, d.column_id);
      if (qc < 0) continue;
      if (!in_time) {
        if (count_stats) atomicAdd(&A.counters[2 + N_BINS], 1ull);
        continue;
      }
      if (A.cols[qc].phys_type != d.phys_type) {
        atomicCAS(A.status, 0, TSKV_ERR_INVALID_ARG);
        continue;
      }
      const uint32_t vclass = (uint32_t)value_class(d.reserved);
      const bool with_time = !((seen_classes >> vclass) & 1);
      seen_classes |= 1u << vclass;
      emit((uint32_t)p, (uint32_t)A.page_bin[p], (uint32_t)qc, with_time, d, !any, tp);
      any = true;
    }
  }
}

// Pass 1: bucket totals + the reader counters.
__global__ void __launch_bounds__(WL_THREADS) k_worklist_count(const WorkListArgs A) {
  extern __shared__ uint32_t s_hist[];  // [N_BINS * n_cols * WL_SUB]
  __shared__ unsigned long long s_pages, s_bytes[N_BINS];
  const uint32_t n_buckets = N_BINS * A.n_cols * WL_SUB;
  for (uint32_t k = threadIdx.x; k < n_buckets; k += WL_THREADS) s_hist[k] = 0;
  if (threadIdx.x == 0) s_pages = 0;
  if (threadIdx.x < N_BINS) s_bytes[threadIdx.x] = 0;
  __syncthreads();
  const uint32_t i = blockIdx.x * WL_THREADS + threadIdx.x;
  if (i < A.n_sel)
    worklist_walk(A, A.walk ? __ldg(A.walk + i) : i, true, [&](uint32_t page, uint32_t bin, uint32_t qc, bool, const tskv_page_desc &d, bool first_in_group, uint32_t tp) {
      atomicAdd(&s_hist[worklist_key(A, page, bin, qc)], 1u);
      // the reader metrics (page_read_count / page_read_bytes) count the time page once per column group
      unsigned long long bytes = d.size, pages = 1;
      if (first_in_group) { bytes += A.descs[tp].size; pages += 1; }
      atomicAdd(&s_bytes[bin], bytes);
      atomicAdd(&s_pages, pages);
    });
  __syncthreads();
  for (uint32_t k = threadIdx.x; k < n_buckets; k += WL_THREADS)
    if (s_hist[k]) atomicAdd(&A.bucket_count[k], s_hist[k]);
  if (threadIdx.x == 0 && s_pages) atomicAdd(&A.counters[0], s_pages);
  if (threadIdx.x < N_BINS && s_bytes[threadIdx.x]) {
    atomicAdd(&A.counters[1], s_bytes[threadIdx.x]);
    atomicAdd(&A.counters[2 + threadIdx.x], s_bytes[threadIdx.x]);
  }
}

// Exclusive offsets of the buckets (bin-major, `per_bin` buckets per bin), bin_cstart, and the cursors reset for pass 2.
// One block.
__global__ void k_worklist_offsets(uint32_t *bucket_count, uint32_t *bucket_off, uint32_t per_bin, uint32_t *bin_cstart) {
  __shared__ uint32_t s_carry;
  __shared__ uint32_t s_warp[32];
  const uint32_t n_buckets = N_BINS * per_bin;
  if (threadIdx.x == 0) s_carry = 0;
  __syncthreads();
  for (uint32_t base = 0; base < n_buckets; base += blockDim.x) {
    const uint32_t k = base + threadIdx.x;
    const uint32_t v = k < n_buckets ? bucket_count[k] : 0;
    uint32_t x = v;
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t y = __shfl_up_sync(FULL, x, o);
      if ((threadIdx.x & 31) >= (uint32_t)o) x += y;
    }
    if ((threadIdx.x & 31) == 31) s_warp[threadIdx.x >> 5] = x;
    __syncthreads();
    if (threadIdx.x < 32) {
      const uint32_t w = threadIdx.x < (blockDim.x >> 5) ? s_warp[threadIdx.x] : 0;
      uint32_t xs = w;
      for (int o = 1; o < 32; o <<= 1) {
        const uint32_t y = __shfl_up_sync(FULL, xs, o);
        if (threadIdx.x >= (uint32_t)o) xs += y;
      }
      s_warp[threadIdx.x] = xs - w;
    }
    __syncthreads();
    const uint32_t excl = s_carry + s_warp[threadIdx.x >> 5] + x - v;
    if (k < n_buckets) {
      bucket_off[k] = excl;
      bucket_count[k] = 0;  // pass 2's cursor
      if (k % per_bin == 0) bin_cstart[k / per_bin] = excl;
    }
    __syncthreads();
    if (threadIdx.x == blockDim.x - 1) s_carry = excl + v;
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    bucket_off[n_buckets] = s_carry;
    bin_cstart[N_BINS] = s_carry;
    bin_cstart[N_BINS + 1] = s_carry;  // total
  }
}

// Pass 2: the same walk; a block reserves its share of every bucket with one atomic and places its items inside it.
__global__ void __launch_bounds__(WL_THREADS) k_worklist_emit(const WorkListArgs A) {
  extern __shared__ uint32_t s_hist[];  // [2][N_BINS * n_cols * WL_SUB]: block counts -> block bases, and the running cursors
  const uint32_t n_buckets = N_BINS * A.n_cols * WL_SUB;
  uint32_t *s_base = s_hist, *s_cur = s_hist + n_buckets;
  for (uint32_t k = threadIdx.x; k < 2 * n_buckets; k += WL_THREADS) s_hist[k] = 0;
  __syncthreads();
  const uint32_t i = blockIdx.x * WL_THREADS + threadIdx.x;
  const uint32_t slot = (i < A.n_sel && A.walk) ? __ldg(A.walk + i) : i;
  if (i < A.n_sel)
    worklist_walk(A, slot, false, [&](uint32_t page, uint32_t bin, uint32_t qc, bool, const tskv_page_desc &, bool, uint32_t) {
      atomicAdd(&s_base[worklist_key(A, page, bin, qc)], 1u);
    });
  __syncthreads();
  for (uint32_t k = threadIdx.x; k < n_buckets; k += WL_THREADS)
    if (s_base[k]) s_base[k] = A.bucket_off[k] + atomicAdd(&A.bucket_count[k], s_base[k]);
  __syncthreads();
  if (i < A.n_sel)
    worklist_walk(A, slot, false, [&](uint32_t page, uint32_t bin, uint32_t qc, bool with_time, const tskv_page_desc &, bool, uint32_t) {
      const uint32_t key = worklist_key(A, page, bin, qc);
      const uint32_t pos = s_base[key] + atomicAdd(&s_cur[key], 1u);
      A.work_page[pos] = page;
      A.work_slot[pos] = slot;
      A.work_qcol[pos] = (uint8_t)(qc | (with_time ? 0x80 : 0));
    });
}

// Host-resident arenas: pull the selected pages over PCIe into the device arena (same offsets).
// One warp per work item, 16-byte coalesced loads from the mapped host range. Replaces the per-series
// file reads of TsmReader::read_adjacent_pages (tsm/reader.rs:236-264).
__global__ void k_gather_pages(const uint8_t *host_arena, uint8_t *dev_arena, const tskv_page_desc *descs,
                               const uint32_t *time_page_of, const uint32_t *work_page,
                               const uint8_t *work_qcol, const uint32_t *bin_cstart, int bin) {
  const uint32_t w0 = bin_cstart[bin], n = bin_cstart[bin + 1];  // the bin's range of the work list
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t warps = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t w = w0 + ((blockIdx.x * blockDim.x + threadIdx.x) >> 5); w < n; w += warps) {
    const uint32_t page = work_page[w];
    const bool with_time = work_qcol[w] & 0x80;
    for (int pass = 0; pass < (with_time ? 2 : 1); pass++) {
      const tskv_page_desc d = descs[pass == 0 ? page : time_page_of[page]];
      const uint4 *src = reinterpret_cast<const uint4 *>(host_arena + d.offset);
      uint4 *dst = reinterpret_cast<uint4 *>(dev_arena + d.offset);
      const uint32_t n16 = d.size >> 4;
      for (uint32_t k = lane; k < n16; k += 32) dst[k] = src[k];
      const uint32_t tail = d.size & 15;
      if (lane < tail) dev_arena[d.offset + (n16 << 4) + lane] = host_arena[d.offset + (n16 << 4) + lane];
    }
  }
}

// Single-block exclusive scan of the per-block counts (n_blocks is small: n_items / 1024).
__global__ void k_scan_blocks(uint32_t *block_count, uint32_t n_blocks, uint32_t *total) {
  __shared__ uint32_t s_warp[32];
  __shared__ uint32_t s_carry;
  if (threadIdx.x == 0) s_carry = 0;
  __syncthreads();
  for (uint32_t base = 0; base < n_blocks; base += blockDim.x) {
    uint32_t i = base + threadIdx.x;
    uint32_t v = i < n_blocks ? block_count[i] : 0;
    uint32_t x = v;
    for (int o = 1; o < 32; o <<= 1) {
      uint32_t y = __shfl_up_sync(FULL, x, o);
      if ((threadIdx.x & 31) >= o) x += y;
    }
    if ((threadIdx.x & 31) == 31) s_warp[threadIdx.x >> 5] = x;
    __syncthreads();
    if (threadIdx.x < 32) {
      uint32_t w = threadIdx.x < (blockDim.x >> 5) ? s_warp[threadIdx.x] : 0;
      uint32_t xs = w;
      for (int o = 1; o < 32; o <<= 1) {
        uint32_t y = __shfl_up_sync(FULL, xs, o);
        if (threadIdx.x >= o) xs += y;
      }
      s_warp[threadIdx.x] = xs - w;  // exclusive warp offsets
    }
    __syncthreads();
    uint32_t excl = s_carry + s_warp[threadIdx.x >> 5] + x - v;
    if (i < n_blocks) block_count[i] = excl;
    __syncthreads();
    if (threadIdx.x == blockDim.x - 1) s_carry = excl + v;
    __syncthreads();
  }
  if (threadIdx.x == 0) *total = s_carry;
}

// Ordered scatter: keeps the kind-sorted order, so the compacted list is still binned by kind;
// bin_cstart[k] = compacted position of the first item of bin k.
__global__ void k_scatter_items(const uint32_t *item_page, const uint32_t *item_cg, uint32_t n_items,
                                const uint8_t *item_flag, const uint32_t *block_offset,
                                const int32_t *cg_slot, const uint32_t *bin_start, uint32_t *work_page,
                                uint32_t *work_slot, uint8_t *work_qcol, uint32_t *bin_cstart,
                                const uint32_t *total) {
  __shared__ uint32_t s_warp[32];
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  uint8_t f = i < n_items ? item_flag[i] : 0;
  uint32_t m = __ballot_sync(FULL, f != 0);
  uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (lane == 0) s_warp[wid] = __popc(m);
  __syncthreads();
  if (threadIdx.x < 32) {
    uint32_t w = threadIdx.x < (blockDim.x >> 5) ? s_warp[threadIdx.x] : 0;
    uint32_t xs = w;
    for (int o = 1; o < 32; o <<= 1) {
      uint32_t y = __shfl_up_sync(FULL, xs, o);
      if (threadIdx.x >= o) xs += y;
    }
    s_warp[threadIdx.x] = xs - w;
  }
  __syncthreads();
  uint32_t pos = block_offset[blockIdx.x] + s_warp[wid] + __popc(m & ((1u << lane) - 1));
  if (i < n_items) {
    if (f) {
      work_page[pos] = item_page[i];
      work_slot[pos] = (uint32_t)cg_slot[item_cg[i]];
      work_qcol[pos] = (uint8_t)(((f & 0x7f) - 1) | (f & 0x80));
    }
    for (int k = 0; k < N_BINS; k++)
      if (bin_start[k] == i) bin_cstart[k] = pos;
  }
  if (i == 0) {
    for (int k = 0; k <= N_BINS; k++)
      if (bin_start[k] >= n_items) bin_cstart[k] = *total;
  }
}

// Page::crc_validation on the device (tskv/src/tsm/page.rs:58-76): CRC-32/IEEE of the data part of every page
// a scan is about to read, checked against the page header. One lane per work item (its field page, plus the
// column group's time page when the item carries it), slicing-by-4 with the tables in shared memory.
// Host-resident arenas run it after the PCIe gather, i.e. on every read like the reference.
__device__ __forceinline__ uint32_t crc_step8(const uint32_t (*t)[256], uint32_t crc, uint32_t lo, uint32_t hi) {
  lo ^= crc;
  return t[7][lo & 0xff] ^ t[6][(lo >> 8) & 0xff] ^ t[5][(lo >> 16) & 0xff] ^ t[4][lo >> 24] ^ t[3][hi & 0xff] ^
         t[2][(hi >> 8) & 0xff] ^ t[1][(hi >> 16) & 0xff] ^ t[0][hi >> 24];
}

__global__ void __launch_bounds__(256)
k_verify_crc(const uint8_t *arena, const tskv_page_desc *descs, const uint32_t *time_page_of,
             const uint32_t *work_page, const uint8_t *work_qcol, const uint32_t *bin_cstart, int bin,
             const uint32_t *crc_tables /* [8][256] */, int32_t *status, unsigned long long *err_page) {
  __shared__ uint32_t s_t[8][256];
  for (uint32_t i = threadIdx.x; i < 2048; i += blockDim.x) s_t[i >> 8][i & 255] = crc_tables[i];
  __syncthreads();
  const uint32_t w0 = bin_cstart[bin], n = bin_cstart[bin + 1];
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t w = w0 + blockIdx.x * blockDim.x + threadIdx.x; w < n; w += stride) {
    const uint32_t page = work_page[w];
    const bool with_time = work_qcol[w] & 0x80;
    for (int pass = 0; pass < (with_time ? 2 : 1); pass++) {
      const uint32_t pg = pass == 0 ? page : time_page_of[page];
      const tskv_page_desc d = descs[pg];
      if (d.size < 16) continue;  // framing errors are reported by the decode kinds
      const uint8_t *p = arena + d.offset;
      const uint32_t bitset_len = load_be32_aligned(p);
      const uint32_t want = load_be32_aligned(p + 12);
      if (16ull + bitset_len > d.size) continue;
      const uint8_t *q = p + 16 + bitset_len;
      uint32_t len = d.size - 16 - bitset_len;
      uint32_t crc = 0xffffffffu;
      while (len && (reinterpret_cast<uintptr_t>(q) & 15)) {  // head bytes up to 16-byte alignment
        crc = (crc >> 8) ^ s_t[0][(crc ^ __ldg(q)) & 0xff];
        q++;
        len--;
      }
      for (; len >= 16; len -= 16, q += 16) {  // one 16-byte load per half sector, slicing-by-8 twice
        const uint4 v = __ldg(reinterpret_cast<const uint4 *>(q));
        crc = crc_step8(s_t, crc, v.x, v.y);
        crc = crc_step8(s_t, crc, v.z, v.w);
      }
      for (; len; len--, q++) crc = (crc >> 8) ^ s_t[0][(crc ^ __ldg(q)) & 0xff];
      if ((crc ^ 0xffffffffu) != want) {
        if (atomicCAS(status, 0, (int)TSKV_ERR_CRC_MISMATCH) == 0) *err_page = pg;
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Row filter of the pushed field predicates (DataFilter, tskv/src/reader/filter.rs:23-142; `column <op> constant`
// joined by AND). One lane per selected column group decodes the group's predicate columns and writes one keep bit per
// row: 1 = every comparison is TRUE. A NULL value, or a group without a page of the column (null-filled by the
// reference, schema_alignmenter.rs:24-44), keeps no row. The fused kernels read the bits next to the validity bitmaps;
// only a bit per row leaves this kernel, never a decoded value.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ bool cmp_true(uint8_t pt, uint8_t op, uint64_t v, uint64_t c) {
  int r;  // -1 / 0 / +1, or 2 for unordered (NaN)
  if (pt == TSKV_PT_I64) r = (int64_t)v < (int64_t)c ? -1 : ((int64_t)v > (int64_t)c ? 1 : 0);
  else if (pt == TSKV_PT_U64) r = v < c ? -1 : (v > c ? 1 : 0);
  else {
    const double a = __longlong_as_double((long long)v), b = __longlong_as_double((long long)c);
    r = (a != a || b != b) ? 2 : (a < b ? -1 : (a > b ? 1 : 0));
  }
  switch (op) {
    case TSKV_CMP_EQ: return r == 0;
    case TSKV_CMP_NE: return r == -1 || r == 1;
    case TSKV_CMP_LT: return r == -1;
    case TSKV_CMP_LE: return r == -1 || r == 0;
    case TSKV_CMP_GT: return r == 1;
    case TSKV_CMP_GE: return r == 1 || r == 0;
    default: return false;
  }
}

__global__ void k_row_filter(const uint8_t *arena, const tskv_page_desc *descs, uint64_t n_descs, const uint32_t *cg_time_page,
                             uint32_t n_cg, const int32_t *cg_slot, const PredicateSet preds, const uint32_t *keep_off,
                             uint32_t *row_keep, int32_t *status, unsigned long long *err_page) {
  const uint32_t cg = blockIdx.x * blockDim.x + threadIdx.x;
  if (cg >= n_cg || cg_slot[cg] < 0) return;
  const uint32_t tp = cg_time_page[cg];
  const uint32_t n_rows = descs[tp].num_values;
  const uint32_t n_words = (n_rows + 31) >> 5;
  uint32_t *keep = row_keep + keep_off[tp];
  for (uint32_t w = 0; w < n_words; w++) keep[w] = 0xffffffffu;
  for (uint32_t k = 0; k < preds.n; k++) {
    const tskv_field_predicate fp = preds.p[k];
    uint64_t pg = 0;
    bool found = false;
    for (uint64_t j = tp + 1; j < n_descs && descs[j].phys_type != TSKV_PT_TIME; j++)
      if (descs[j].column_id == fp.column_id) { pg = j; found = true; break; }
    if (!found) {  // the column is NULL for every row of this group
      for (uint32_t w = 0; w < n_words; w++) keep[w] = 0;
      continue;
    }
    const tskv_page_desc d = descs[pg];
    tskv_status st = d.phys_type != fp.phys_type ? TSKV_ERR_INVALID_ARG : kind_status(d.reserved);
    if (st == TSKV_OK) {
      PageView pv;
      pv.open(arena, d);
      BitCursor bits;
      bits.init(pv.bitset);
      AnyCursor<> cur;
      st = cur.open(pv, d.reserved);
      const bool allnull = d.reserved == DK_ALLNULL;
      uint32_t word = 0;
      for (uint32_t r = 0; r < n_rows && st == TSKV_OK; r++) {
        const bool valid = bits.next(r) && !allnull;
        bool pass = false;
        if (valid) {
          const uint64_t v = cur.next();
          if (cur.failed()) { st = cur.stream_error() ? TSKV_ERR_SHORT_BLOCK : TSKV_ERR_BITSET_MISMATCH; break; }
          pass = cmp_true(fp.phys_type, fp.op, v, fp.value);
        } else if (r == 0 && !cur.is_gorilla) {
          cur.d.skip_first_if_s8b_sc();
        }
        word |= (pass ? 1u : 0u) << (r & 31);
        if ((r & 31) == 31 || r == n_rows - 1) { keep[r >> 5] &= word; word = 0; }
      }
      if (st == TSKV_OK && cur.is_gorilla && cur.g.consumed_any() && !cur.g.drain()) st = TSKV_ERR_SHORT_BLOCK;
    }
    if (st != TSKV_OK && atomicCAS(status, 0, (int)st) == 0) *err_page = pg;
  }
}

// ------------------------------------------------------------------------------------------------
// fused scan
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ bool cas128(unsigned long long *addr, unsigned long long cmp_lo,
                                       unsigned long long cmp_hi, unsigned long long new_lo,
                                       unsigned long long new_hi, unsigned long long *old_lo,
                                       unsigned long long *old_hi) {
  unsigned long long olo, ohi;
  asm volatile(
      "{\n\t.reg .b128 c, v, o;\n\t"
      "mov.b128 c, {%2, %3};\n\t"
      "mov.b128 v, {%4, %5};\n\t"
      "atom.global.relaxed.gpu.cas.b128 o, [%6], c, v;\n\t"
      "mov.b128 {%0, %1}, o;\n\t}"
      : "=l"(olo), "=l"(ohi)
      : "l"(cmp_lo), "l"(cmp_hi), "l"(new_lo), "l"(new_hi), "l"(addr)
      : "memory");
  *old_lo = olo;
  *old_hi = ohi;
  return olo == cmp_lo && ohi == cmp_hi;
}

// pair = {i64 key, u64 val}; keep the pair with the smaller (IS_MIN) / larger key.
template <bool IS_MIN>
__device__ __forceinline__ void atomic_select_pair(uint64_t *pair, int64_t key, uint64_t val) {
  unsigned long long *p = reinterpret_cast<unsigned long long *>(pair);
  unsigned long long cur_k = IS_MIN ? 0x7fffffffffffffffull : 0x8000000000000000ull;  // identity
  unsigned long long cur_v = 0;
  for (;;) {
    bool better = IS_MIN ? key < (int64_t)cur_k : key > (int64_t)cur_k;
    if (!better) return;
    unsigned long long ok, ov;
    if (cas128(p, cur_k, cur_v, (unsigned long long)key, val, &ok, &ov)) return;
    cur_k = ok;
    cur_v = ov;
  }
}

// Ordered i64 key of a value of physical type pt (signed compare == typed compare; f64: IEEE
// totalOrder).
__device__ __forceinline__ int64_t okey(uint64_t v, uint8_t pt) {
  uint64_t flip = pt == TSKV_PT_U64 ? 0x8000000000000000ull
                  : pt == TSKV_PT_F64 ? (uint64_t)(((int64_t)v >> 63) & 0x7fffffffffffffffll)
                                      : 0ull;
  return (int64_t)(v ^ flip);
}
__host__ __device__ inline uint64_t okey_inv(int64_t k, uint8_t pt) {
  uint64_t v = (uint64_t)k;
  if (pt == TSKV_PT_U64) return v ^ 0x8000000000000000ull;
  if (pt == TSKV_PT_F64) return v ^ (uint64_t)((k >> 63) & 0x7fffffffffffffffll);
  return v;
}

__device__ __forceinline__ uint64_t shfl_u64(uint64_t v, int src) {
  return ((uint64_t)__shfl_sync(FULL, (uint32_t)(v >> 32), src) << 32) |
         __shfl_sync(FULL, (uint32_t)v, src);
}
__device__ __forceinline__ uint64_t shfl_xor_u64(uint64_t v, int m) {
  return ((uint64_t)__shfl_xor_sync(FULL, (uint32_t)(v >> 32), m) << 32) |
         __shfl_xor_sync(FULL, (uint32_t)v, m);
}

// Integer sum: the low word is the reference's wrapping i64/u64 SUM; with MEAN the carries go to a high
// word so that mean = exact 128-bit sum / count (DataFusion's avg accumulates in f64 and never wraps).
__device__ __forceinline__ void add_int_sum(uint64_t *sum_cell, uint64_t *hi_cell, uint8_t mask, uint64_t lo, int64_t hi) {
  unsigned long long *plo = reinterpret_cast<unsigned long long *>(sum_cell);
  if (mask & TSKV_AGG_MEAN) {
    unsigned long long old = atomicAdd(plo, (unsigned long long)lo);
    hi += (old + lo < old) ? 1 : 0;
    if (hi) atomicAdd(reinterpret_cast<unsigned long long *>(hi_cell), (unsigned long long)hi);
  } else {
    atomicAdd(plo, (unsigned long long)lo);
  }
}

// count / sum / min / max of one run into the partial table: `tab` is either the global state (offsets
// *_off) or the CTA's shared-memory table (offsets s_*).
__device__ __forceinline__ void table_update(const ScanParams &P, uint64_t *stab, const ColState &cs, uint64_t cell,
                                             uint8_t mask, bool f64, uint32_t cnt, uint64_t sum, int64_t shi,
                                             int64_t kmin, int64_t kmax) {
  const bool sm = P.use_smem != 0;
  uint64_t *tab = sm ? stab : P.state;
  atomicAdd(reinterpret_cast<unsigned long long *>(tab + (sm ? cs.s_count : cs.count_off) + cell), (unsigned long long)cnt);
  if (mask & (TSKV_AGG_SUM | TSKV_AGG_MEAN)) {
    uint64_t *sc = tab + (sm ? cs.s_sum : cs.sum_off) + cell;
    if (f64) atomicAdd(reinterpret_cast<double *>(sc), __longlong_as_double((long long)sum));
    else add_int_sum(sc, tab + (sm ? cs.s_hi : cs.sumhi_off) + cell, mask, sum, shi);
  }
  if (mask & TSKV_AGG_MIN) atomicMin(reinterpret_cast<long long *>(tab + (sm ? cs.s_min : cs.min_off) + cell), (long long)kmin);
  if (mask & TSKV_AGG_MAX) atomicMax(reinterpret_cast<long long *>(tab + (sm ? cs.s_max : cs.max_off) + cell), (long long)kmax);
}

// Warp reductions on REDUX (one instruction per 32-bit word instead of a 5-step shuffle butterfly).
// max / min of signed 64-bit values: reduce the high words, then the low words of the lanes that tie.
__device__ __forceinline__ int64_t warp_max_i64(int64_t v) {
  const int32_t hi = (int32_t)(v >> 32);
  const int32_t mh = __reduce_max_sync(FULL, hi);
  const uint32_t lo = hi == mh ? (uint32_t)v : 0u;
  const uint32_t ml = __reduce_max_sync(FULL, lo);
  return (int64_t)(((uint64_t)(uint32_t)mh << 32) | ml);
}
__device__ __forceinline__ int64_t warp_min_i64(int64_t v) {
  const int32_t hi = (int32_t)(v >> 32);
  const int32_t mh = __reduce_min_sync(FULL, hi);
  const uint32_t lo = hi == mh ? (uint32_t)v : 0xffffffffu;
  const uint32_t ml = __reduce_min_sync(FULL, lo);
  return (int64_t)(((uint64_t)(uint32_t)mh << 32) | ml);
}
// Wrapping sum of 32 u64 values plus the carries out of bit 63 (three 22-bit limbs; 32 * 2^22 < 2^32).
__device__ __forceinline__ uint64_t warp_sum_u64(uint64_t v, uint32_t *carry) {
  const uint32_t s0 = __reduce_add_sync(FULL, (uint32_t)v & 0x3fffffu);
  const uint32_t s1 = __reduce_add_sync(FULL, (uint32_t)(v >> 22) & 0x3fffffu);
  const uint32_t s2 = __reduce_add_sync(FULL, (uint32_t)(v >> 44));  // 20 bits
  const uint64_t low = (uint64_t)s0 + ((uint64_t)s1 << 22);           // < 2^50
  const uint64_t top = (uint64_t)s2 + (low >> 44);                     // units of 2^44, < 2^26
  *carry = (uint32_t)(top >> 20);
  return (low & 0xfffffffffffull) | (top << 44);
}

// Partial aggregate of one (page, bucket) run, held in registers by one lane.
struct RunAcc {
  uint32_t count;
  uint64_t sum;      // i64 wrapping sum bits, or f64 sum bits
  int64_t sum_hi;    // high word of the exact integer sum (only maintained for MEAN on int columns)
  int64_t kmin, kmax;
  int64_t first_ts, last_ts;
  uint64_t first_val, last_val;
  bool first_ok, last_ok;  // the run's min/max-time row had a non-null value (first.rs:91-94)
};

struct ScanCtx {
  const ScanParams *P;
};

// Warp-converged flush of run partials into the global state. `active` lanes carry a finished
// run for cell `gcell` (= qcol * n_cells + cell). When every flushing lane targets the same cell
// (the common lock-step case of GROUP BY bucket) the partials are combined with a butterfly first
// and one lane issues the atomics.
template <bool SEL>
__device__ __forceinline__ void warp_flush(const ScanParams &P, uint64_t *stab, bool active, uint32_t qcol,
                                           uint64_t cell, int64_t bucket, uint8_t pt, uint8_t mask,
                                           RunAcc &a, uint32_t slot) {
  uint32_t m = __ballot_sync(FULL, active);
  if (m == 0) return;
  const uint64_t gcell = (uint64_t)qcol * P.n_cells + cell;
  int leader = __ffs(m) - 1;
  uint64_t lcell = shfl_u64(gcell, leader);
  bool same = __all_sync(FULL, !active || gcell == lcell);
  // first/last keys (only meaningful on active lanes)
  int64_t kf = a.first_ts, kl = a.last_ts;
  if (SEL && P.slot_bits) {
    // rel > 0 by construction (see ScanParams); the host checked rel_bits + slot_bits <= 62
    uint64_t base = P.width > 0 ? (uint64_t)P.first_bucket_start + (uint64_t)(bucket - 1) * (uint64_t)P.width
                                : (uint64_t)P.rel_base;
    kf = (int64_t)((((uint64_t)a.first_ts - base) << P.slot_bits) | slot);
    kl = (int64_t)((((uint64_t)a.last_ts - base) << P.slot_bits) | (P.slot_max - slot));
  }
  const bool is_f64 = (uint8_t)__shfl_sync(FULL, (uint32_t)pt, leader) == TSKV_PT_F64;
  const bool own_f64 = pt == TSKV_PT_F64;
  if (same && __popc(m) > 1) {
    const uint32_t cnt = active ? a.count : 0;
    uint64_t sum = active ? a.sum : 0;  // 0 bits == +0.0
    int64_t shi = active ? a.sum_hi : 0;
    const uint32_t tot = __reduce_add_sync(FULL, cnt);
    int64_t kmin = INT64_MAX, kmax = INT64_MIN, fk = INT64_MAX, lk = INT64_MIN;
    if (tot) {  // warp-uniform
      if (is_f64) {
        double d = __longlong_as_double((long long)sum);
        for (int o = 16; o; o >>= 1) d += __longlong_as_double((long long)shfl_xor_u64((uint64_t)__double_as_longlong(d), o));
        sum = (uint64_t)__double_as_longlong(d);
      } else {
        uint32_t carry;
        sum = warp_sum_u64(sum, &carry);
        shi = (int64_t)(int32_t)__reduce_add_sync(FULL, (uint32_t)shi) + carry;  // |per-lane hi| < 2^26
      }
      const uint32_t lmask = __shfl_sync(FULL, (uint32_t)mask, leader);  // same cell => same column => same mask
      if (lmask & TSKV_AGG_MIN) kmin = warp_min_i64((active && a.count) ? a.kmin : INT64_MAX);
      if (lmask & TSKV_AGG_MAX) kmax = warp_max_i64((active && a.count) ? a.kmax : INT64_MIN);
    }
    if (SEL) {
      fk = warp_min_i64((active && a.first_ok) ? kf : INT64_MAX);
      lk = warp_max_i64((active && a.last_ok) ? kl : INT64_MIN);
    }
    // owners of the winning first / last keys supply the values
    uint32_t mf = 0, ml = 0;
    uint64_t fv = 0, lv = 0;
    if (SEL) {
      mf = __ballot_sync(FULL, active && a.first_ok && kf == fk);
      ml = __ballot_sync(FULL, active && a.last_ok && kl == lk);
      fv = shfl_u64(a.first_val, mf ? __ffs(mf) - 1 : 0);
      lv = shfl_u64(a.last_val, ml ? __ffs(ml) - 1 : 0);
    }
    if ((int)(threadIdx.x & 31) == leader) {
      const ColState &cs = P.cols[qcol];
      uint64_t *st = P.state;
      if (tot) table_update(P, stab, cs, cell, mask, is_f64, tot, sum, shi, kmin, kmax);
      if (SEL && (mask & TSKV_AGG_FIRST) && mf) atomic_select_pair<true>(st + cs.first_off + 2 * cell, fk, fv);
      if (SEL && (mask & TSKV_AGG_LAST) && ml) atomic_select_pair<false>(st + cs.last_off + 2 * cell, lk, lv);
    }
  } else if (active) {
    const ColState &cs = P.cols[qcol];
    uint64_t *st = P.state;
    if (a.count) table_update(P, stab, cs, cell, mask, own_f64, a.count, a.sum, a.sum_hi, a.kmin, a.kmax);
    if (SEL && (mask & TSKV_AGG_FIRST) && a.first_ok) atomic_select_pair<true>(st + cs.first_off + 2 * cell, kf, a.first_val);
    if (SEL && (mask & TSKV_AGG_LAST) && a.last_ok) atomic_select_pair<false>(st + cs.last_off + 2 * cell, kl, a.last_val);
  }
}

__device__ __forceinline__ void report_error(const ScanParams &P, tskv_status st, uint32_t page) {
  if (atomicCAS(P.status, 0, (int)st) == 0) *P.err_page = page;
}

// Bucket bookkeeping of one lane: timestamps in [lo, hi] (inclusive) map to bucket `idx`.
struct BucketState {
  int64_t lo, hi;
  uint32_t idx;
  bool valid;
  bool floor_regime;  // dividend >= 0: the bucket is [start, start + w)
};

// `sliding_window(t, w, w, origin, 0)` (time_window.rs:184-198): start = t - ((t - o + w) % w) with
// truncating %, so for a negative dividend the window is (start - w, start] (kept as-is).
__device__ __forceinline__ bool locate_bucket(const ScanParams &P, int64_t t, BucketState &b) {
  if (P.width <= 0) {
    b.lo = INT64_MIN; b.hi = INT64_MAX; b.idx = 0; b.valid = true; b.floor_regime = false;
    return true;
  }
  const int64_t w = P.width;
  // the last t whose dividend t - origin_mod + w does not wrap: floor-regime buckets end there, rows past it belong to
  // the reference's wrapped windows
  const int64_t cap = P.floor_cap;
  if (b.valid && b.floor_regime && t > b.hi && (uint64_t)t - (uint64_t)b.hi <= (uint64_t)w && t <= cap &&
      b.idx + 1 < P.n_buckets) {  // next bucket of the floor-aligned regime
    b.lo = b.hi + 1;
    b.hi = (int64_t)((uint64_t)b.hi + ((uint64_t)cap - (uint64_t)b.hi < (uint64_t)w ? (uint64_t)cap - (uint64_t)b.hi : (uint64_t)w));
    b.idx += 1;
    return true;
  }
  int64_t dividend = (int64_t)((uint64_t)t - (uint64_t)P.origin_mod + (uint64_t)w);
  int64_t rem = dividend % w;
  int64_t start = (int64_t)((uint64_t)t - (uint64_t)rem);
  int64_t diff = (int64_t)((uint64_t)start - (uint64_t)P.first_bucket_start);
  if (diff < 0 || diff % w != 0 || diff / w >= (int64_t)P.n_buckets) return false;
  b.idx = (uint32_t)(diff / w);
  // rows below wrap_lo (dividend wrapped downwards, >= 0) share a start up to wrap_lo - 1 at most, and the next bucket is
  // not start + w: they take no step
  const bool wrapped = t < P.wrap_lo;
  if (dividend >= 0) {  // [start, start + w), cut at cap (start <= t <= cap)
    const uint64_t room = (uint64_t)(wrapped ? P.wrap_lo - 1 : cap) - (uint64_t)start;
    b.lo = start;
    b.hi = (int64_t)((uint64_t)start + (room < (uint64_t)(w - 1) ? room : (uint64_t)(w - 1)));
  } else {  // (start - w, start], cut at wrap_lo
    b.lo = start - w + 1; b.hi = start;
    if (b.lo < P.wrap_lo) b.lo = P.wrap_lo;
  }
  b.floor_regime = dividend >= 0 && !wrapped;
  b.valid = true;
  return true;
}

// Closed time ranges (TimeRange::contains, predicate/domain.rs:95-98): is t selected, and over which
// inclusive interval [lo, hi] around t does that answer stay the same?
__device__ __forceinline__ bool range_span(const ScanParams &P, int64_t t, int64_t &lo, int64_t &hi) {
  lo = INT64_MIN;
  hi = INT64_MAX;
  if (P.n_ranges == 0) return true;
  if (P.n_ranges == 1) {  // the common single BETWEEN
    const int64_t a = P.ranges[0].min_ts, b = P.ranges[0].max_ts;
    if (t < a) { hi = a - 1; return false; }
    if (t > b) { lo = b + 1; return false; }
    lo = a; hi = b;
    return true;
  }
  bool in = false;
#pragma unroll 1
  for (uint32_t k = 0; k < P.n_ranges; k++) {
    const int64_t a = P.ranges[k].min_ts, b = P.ranges[k].max_ts;
    if (t >= a && t <= b) {
      if (!in) { lo = a; hi = b; in = true; }
    } else if (!in) {
      if (a > t && a - 1 < hi) hi = a - 1;
      if (b < t && a <= b && b + 1 > lo) lo = b + 1;
    }
  }
  return in;
}

// Like range_span for a tombstone list: is t inside one of the n closed ranges, and narrow [lo, hi] to an interval
// around t over which that answer holds.
__device__ __forceinline__ bool tomb_span(const tskv_time_range *r, uint32_t n, int64_t t, int64_t &lo, int64_t &hi) {
  bool in = false;
  int64_t l = INT64_MIN, h = INT64_MAX;
#pragma unroll 1
  for (uint32_t k = 0; k < n; k++) {
    const int64_t a = r[k].min_ts, b = r[k].max_ts;
    if (a > b) continue;
    if (t >= a && t <= b) {
      if (!in) { l = a; h = b; in = true; }
    } else if (!in) {
      if (a > t && a - 1 < h) h = a - 1;
      if (b < t && b + 1 > l) l = b + 1;
    }
  }
  lo = lo > l ? lo : l;
  hi = hi < h ? hi : h;
  return in;
}

// Tombstone lists of one field page: .x/.y = offset/count of the series' row-drop ranges, .z/.w = of the
// (series, column) null-mask ranges (binary search in the sorted keys, once per page).
__device__ __forceinline__ uint4 tomb_lookup(const ScanParams &P, uint32_t series, uint32_t column) {
  uint4 out = make_uint4(0, 0, 0, 0);
#pragma unroll 1
  for (int pass = 0; pass < 2; pass++) {
    const uint64_t key = ((uint64_t)series << 32) | (pass == 0 ? (uint64_t)TSKV_TOMB_ALL : (uint64_t)column);
    uint32_t lo = 0, hi = P.n_tomb_keys;
    while (lo < hi) {
      const uint32_t mid = (lo + hi) >> 1;
      if (__ldg(P.tomb_keys + mid) < key) lo = mid + 1;
      else hi = mid;
    }
    if (lo < P.n_tomb_keys && __ldg(P.tomb_keys + lo) == key) {
      const uint32_t a = __ldg(P.tomb_off + lo), b = __ldg(P.tomb_off + lo + 1);
      if (pass == 0) { out.x = a; out.y = b - a; }
      else { out.z = a; out.w = b - a; }
    }
  }
  return out;
}

// One chunk of <= 32 work items, one lane per field page. The whole warp stays converged; lanes
// without a page (or past their last row) idle through the loop. Generic path (time pages with NULLs or raw / unusual
// time encodings - nothing the reference's writer produces): row by row, streams read straight from global memory.
// SEL: the query wants FIRST/LAST somewhere (tracks the (ts, value) of each run's end rows).
template <int TK, int VK, bool SEL>
__device__ __forceinline__ void scan_chunk_rows(const ScanParams &P, uint32_t item_begin, uint32_t item_end,
                                             uint32_t /*ring_base*/, uint64_t *stab, uint4 *s_tomb) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t item = item_begin + lane;
  const bool have_item = item < item_end;
  const uint32_t tslot = 0, vslot = 0;

  uint32_t page = 0, slot = 0, qcol = 0, n_rows = 0;
  uint8_t pt = TSKV_PT_I64, mask = 0;
  PageView tpv, vpv;
  BitCursor tbits, vbits;
  DeltaCursor<TK == TK_RLE ? DK_RLE_SC : TK == TK_S8B ? DK_S8B_SC : -1, BeStream> tcur;
  DeltaCursor<VK == VK_S8B ? DK_S8B_ZZ : -1, BeStream> vcur_d;
  GorillaCursor<BeStream> vcur_g;
  bool allnull = false;
  const uint32_t *keepw = nullptr;  // row-filter keep bits of the column group (k_row_filter), or null
  uint32_t kword = 0xffffffffu;

  if (have_item) {
    page = P.work_page[item];
    slot = P.work_slot[item];
    qcol = P.work_qcol[item] & 0x7f;
    const tskv_page_desc vd = P.descs[page];
    const uint32_t tpage = P.time_page_of[page];
    const tskv_page_desc td = P.descs[tpage];
    if (P.row_keep) keepw = P.row_keep + P.keep_off[tpage];
    pt = P.cols[qcol].phys_type;
    mask = P.cols[qcol].agg_mask;
    if (P.has_tomb) s_tomb[threadIdx.x] = tomb_lookup(P, vd.series_id, vd.column_id);
    tskv_status st = kind_status(td.reserved);
    if (st == TSKV_OK) st = kind_status(vd.reserved);
    if (st != TSKV_OK) {
      report_error(P, st, st == kind_status(td.reserved) ? tpage : page);
    } else {
      tpv.open(P.arena, td);
      vpv.open(P.arena, vd);
      n_rows = vd.num_values;
      tbits.init(tpv.bitset);
      vbits.init(vpv.bitset);
      st = tcur.open(tpv, td.reserved, tslot);
      if (st == TSKV_OK) {
        if (VK == VK_GOR) st = vcur_g.open(vpv, vslot);
        else { st = vcur_d.open(vpv, vd.reserved, vslot); allnull = vd.reserved == DK_ALLNULL; }
      }
      if (st != TSKV_OK) { report_error(P, st, page); n_rows = 0; }
      if (td.reserved == DK_ALLNULL) n_rows = 0;  // no time values: every row fails is_not_null(time)
    }
  }

  RunAcc acc;
  acc.count = 0; acc.sum = 0; acc.sum_hi = 0; acc.kmin = INT64_MAX; acc.kmax = INT64_MIN;
  acc.first_ts = acc.last_ts = 0; acc.first_val = acc.last_val = 0; acc.first_ok = acc.last_ok = false;
  BucketState bk; bk.valid = false; bk.floor_regime = false; bk.lo = 0; bk.hi = 0; bk.idx = 0;
  bool have_run = false;
  uint32_t run_idx = 0;
  uint32_t row = 0;
  uint32_t n_points = 0, n_inrange = 0;
  const bool is_f64 = pt == TSKV_PT_F64;
  const bool mean_hi = !is_f64 && (mask & TSKV_AGG_MEAN);

  for (;;) {
    const bool has = row < n_rows;
    if (!__any_sync(FULL, has || have_run)) break;
    bool flush = false, inr = false, vv = false, newrun = false;
    int64_t t = 0;
    uint64_t v = 0;
    if (has) {
      const bool tv = tbits.next(row);
      vv = vbits.next(row) && !allnull;
      bool ok = true;
      if (tv) { t = (int64_t)tcur.next(); ok = !tcur.exhausted; }
      else if (row == 0) tcur.skip_first_if_s8b_sc();
      if (!ok) { report_error(P, TSKV_ERR_BITSET_MISMATCH, P.time_page_of[page]); n_rows = 0; }
      if (vv && ok) {
        v = VK == VK_GOR ? vcur_g.next() : vcur_d.next();
        ok = VK == VK_GOR ? !vcur_g.done : !vcur_d.exhausted;
        if (!ok) {
          report_error(P, (VK == VK_GOR && vcur_g.err) ? TSKV_ERR_SHORT_BLOCK : TSKV_ERR_BITSET_MISMATCH, page);
          n_rows = 0;
        } else {
          n_points++;
        }
      }
      if (keepw && (row & 31) == 0) kword = __ldg(keepw + (row >> 5));
      const bool kept = (kword >> (row & 31)) & 1;  // the row filter (DataFilter) drops the row like the time ranges do
      row++;
      if (ok && tv && kept) {
        inr = P.n_ranges == 0;
#pragma unroll 1
        for (uint32_t k = 0; k < P.n_ranges && !inr; k++) inr = t >= P.ranges[k].min_ts && t <= P.ranges[k].max_ts;
        if (P.has_tomb && inr) {  // decode_pages' tombstone handling, row by row (reader.rs:507-551)
          const uint4 tl = s_tomb[threadIdx.x];
          int64_t lo = INT64_MIN, hi = INT64_MAX;
          if (tomb_span(P.tomb_ranges, P.n_tomb_global, t, lo, hi) || tomb_span(P.tomb_ranges + tl.x, tl.y, t, lo, hi)) inr = false;
          else if (tomb_span(P.tomb_ranges + tl.z, tl.w, t, lo, hi)) vv = false;
        }
      }
      if (inr) {
        n_inrange++;
        bool same_bucket = bk.valid && t >= bk.lo && t <= bk.hi;
        if (!same_bucket) {
          if (!locate_bucket(P, t, bk)) {
            report_error(P, TSKV_ERR_BUCKET_RANGE, page);
            inr = false;
            bk.valid = false;
          }
        }
        if (inr && (!have_run || bk.idx != run_idx)) { newrun = true; flush = have_run; }
      }
    } else {
      flush = have_run;
    }
    warp_flush<SEL>(P, stab, flush, qcol, group_cell_base(P, slot) + run_idx, (int64_t)run_idx, pt, mask, acc, slot);
    if (flush) have_run = false;
    if (has && inr) {
      if (newrun) {
        have_run = true;
        run_idx = bk.idx;
        acc.count = 0; acc.sum = 0; acc.sum_hi = 0; acc.kmin = INT64_MAX; acc.kmax = INT64_MIN;
        if (SEL) {
          acc.first_ts = acc.last_ts = t;
          acc.first_val = acc.last_val = v;
          acc.first_ok = acc.last_ok = vv;
        }
      } else if (SEL) {
        if (t < acc.first_ts) { acc.first_ts = t; acc.first_val = v; acc.first_ok = vv; }
        if (t > acc.last_ts) { acc.last_ts = t; acc.last_val = v; acc.last_ok = vv; }
      }
      if (vv) {
        acc.count++;
        if (is_f64) acc.sum = (uint64_t)__double_as_longlong(__longlong_as_double((long long)acc.sum) + __longlong_as_double((long long)v));
        else {
          acc.sum += v;
          if (mean_hi) acc.sum_hi += (acc.sum < v ? 1 : 0) + (pt == TSKV_PT_I64 ? ((int64_t)v >> 63) : 0);
        }
        int64_t k = okey(v, pt);
        acc.kmin = k < acc.kmin ? k : acc.kmin;
        acc.kmax = k > acc.kmax ? k : acc.kmax;
      }
    }
  }
  // The reference decodes a gorilla page to its sentinel (float.rs:480-591): a stream that ends
  // without one is an error even when enough values were produced.
  if (VK == VK_GOR && have_item && n_rows != 0 && vcur_g.consumed_any() && !vcur_g.drain())
    report_error(P, TSKV_ERR_SHORT_BLOCK, page);
  // statistics
  n_points = __reduce_add_sync(FULL, n_points);
  n_inrange = __reduce_add_sync(FULL, n_inrange);
  if (lane == 0) {
    if (n_points) atomicAdd(&P.stats[0], (unsigned long long)n_points);
    if (n_inrange) atomicAdd(&P.stats[1], (unsigned long long)n_inrange);
  }
}

// Segment-wise variant for time pages without nulls (every reference-written page: flush rejects a
// time column with nulls, mem_cache/series_data.rs:303-340) - the fast path. Per lane:
//   1. a lean look-ahead loop over the TIMESTAMPS finds the next segment = maximal run of rows whose
//      (selected by the time ranges, bucket) is the same;
//   2. the warp flushes finished runs (converged, once per segment instead of once per row);
//   3. a tight loop decodes the segment's VALUES and accumulates them in registers, one validity-bitmap
//      word (<= 32 rows) at a time with an all-valid fast path.
// Rows of a page are time-sorted (tsm/chunk.rs:100-110), so the first / last row of a run carry its
// min / max timestamp (what first()/last() pick with sort_to_indices, first.rs:139-148).
template <int VK>
struct ValueAcc {  // count / sum / min / max of one run; VK fixes the arithmetic at compile time
  uint32_t count;
  uint64_t sum;    // f64: the sum's bits. Integers, while accumulating: sum of the values' LOW 32-bit halves
  int64_t sum_hi;  // integers, while accumulating: sum of the HIGH halves (sign- / zero-extended); see fold()
  int64_t kmin, kmax;
  // Narrow runs (add32: integer values that sign-extend from their low 32 bits) keep `sum` = the exact 64-bit sum of the
  // values (|sum| < 2^63 for 2^32 rows) and the 32-bit min / max in the LOW words of kmin / kmax; fold(pt, true) turns
  // them into the wide run's (sum, sum_hi, keys). A run is narrow or wide from reset to fold.
  __device__ __forceinline__ void reset(bool narrow = false) {
    count = 0; sum = 0; sum_hi = 0;
    kmin = narrow ? INT32_MAX : INT64_MAX;
    kmax = narrow ? INT32_MIN : INT64_MIN;
  }
  __device__ __forceinline__ static int64_t with_lo(int64_t x, int32_t lo) {
    return (int64_t)(((uint64_t)x & 0xffffffff00000000ull) | (uint32_t)lo);
  }
  __device__ __forceinline__ void add32(uint32_t v) {
    sum += (uint64_t)(int64_t)(int32_t)v;
    kmin = with_lo(kmin, min((int32_t)kmin, (int32_t)v));
    kmax = with_lo(kmax, max((int32_t)kmax, (int32_t)v));
  }
  // pt / flip are per-lane constants (flip = okey's xor mask for integer columns).
  // Integer sums are kept as two 64-bit accumulators of 32-bit halves: exact for 2^32 rows without any carry
  // bookkeeping per value (the wrapping SUM and the exact 128-bit sum MEAN needs both fall out of fold()).
  __device__ __forceinline__ void add(uint64_t v, uint8_t pt, uint64_t flip, bool /*mean_hi*/ = false) {
    int64_t key;
    if (VK == VK_GOR || (VK == VK_GEN && pt == TSKV_PT_F64)) {
      sum = (uint64_t)__double_as_longlong(__longlong_as_double((long long)sum) + __longlong_as_double((long long)v));
      key = (int64_t)(v ^ (uint64_t)(((int64_t)v >> 63) & 0x7fffffffffffffffll));
    } else {
      sum += (uint32_t)v;
      sum_hi += pt == TSKV_PT_I64 ? (int64_t)(int32_t)(v >> 32) : (int64_t)(v >> 32);
      key = (int64_t)(v ^ flip);
    }
    kmin = key < kmin ? key : kmin;
    kmax = key > kmax ? key : kmax;
  }
  // End of the run: integers -> (sum, sum_hi) = low / high word of the exact 128-bit sum (sum = the reference's wrapping
  // i64 / u64 SUM). Call once, right before the partial is handed to a flush.
  __device__ __forceinline__ void fold(uint8_t pt, bool narrow = false) {
    if (VK == VK_GOR || (VK == VK_GEN && pt == TSKV_PT_F64)) return;
    if (narrow) {  // u64 values of a narrow run lie in [0, 2^31): their sum is >= 0 like the i64 sign extension says
      const uint64_t flip = pt == TSKV_PT_U64 ? 0x8000000000000000ull : 0ull;
      sum_hi = (int64_t)sum >> 63;
      kmin = (int64_t)((uint64_t)(int64_t)(int32_t)kmin ^ flip);
      kmax = (int64_t)((uint64_t)(int64_t)(int32_t)kmax ^ flip);
      return;
    }
    const uint64_t x = (uint64_t)sum_hi << 32;
    const uint64_t lo = x + sum;
    sum_hi = (pt == TSKV_PT_I64 ? (sum_hi >> 32) : (int64_t)((uint64_t)sum_hi >> 32)) + (lo < x ? 1 : 0);
    sum = lo;
  }
};

// ------------------------------------------------------------------------------------------------
// Staged flush (GROUP BY bucket, no FIRST/LAST). The 32 pages of a warp usually cross a bucket boundary at the same
// row (TSBS-aligned timestamps), so all lanes finish a run for the SAME cell at the same time. Combining 32 partials
// with warp reductions (REDUX / butterflies) and then updating the shared table with CAS-loop atomics costs ~230
// instructions per 6-row segment. Instead every lane parks its partial in a per-warp staging area
//   stage[slot][quantity][lane]          (one conflict-free STS.64 per quantity)
// and every NS flushes the warp reduces the parked partials TRANSPOSED: lane j owns slot j % NS and sums the partials
// of NS source lanes serially (every lane does useful work on every instruction), xor-shuffle steps combine the 32 / NS
// lane groups, and NS lanes update the CTA table.
// NS = flush_slots(TK) slots per warp: 4 (5 152 bytes) for the RLE-timestamp kernels, 2 (2 576 bytes) for the
// simple8b-timestamp kernels, whose two staging rings per warp would otherwise keep them at 3 CTAs per SM. A jittered
// simple8b time page flushes about once per bucket after a few hundred instructions per row, so the extra reduce pass
// per two flushes costs little there. Building with -DTSKV_FLUSH_SLOTS=n gives every kernel n slots.
// ------------------------------------------------------------------------------------------------
#ifdef TSKV_FLUSH_SLOTS
constexpr int FLUSH_SLOTS = TSKV_FLUSH_SLOTS;
__host__ __device__ constexpr int flush_slots(int /*tk*/) { return FLUSH_SLOTS; }
#else
constexpr int FLUSH_SLOTS = 4;
__host__ __device__ constexpr int flush_slots(int tk) { return tk == TK_S8B ? 2 : FLUSH_SLOTS; }
#endif
constexpr int FLUSH_Q = 5;  // count | sum | sum_hi | min key | max key
__host__ __device__ constexpr uint32_t flush_stage_bytes(int ns) { return (ns * FLUSH_Q * 32 + ns) * 8; }  // + one meta word per slot

template <int VK, int NS>
__device__ __forceinline__ void reduce_staged(const ScanParams &P, uint64_t *stab, uint64_t *stage, uint32_t n_slots) {
  __syncwarp();
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t s = lane & (NS - 1), g = lane / NS;
  const uint64_t meta = stage[NS * FLUSH_Q * 32 + s];  // (query column << 32) | cell
  const uint32_t qcol = (uint32_t)(meta >> 32);
  const ColState &cs = P.cols[s < n_slots ? qcol : 0];
  const bool is_f64 = VK == VK_GOR || (VK == VK_GEN && cs.phys_type == TSKV_PT_F64);
  uint64_t cnt = 0, sum = 0;
  int64_t hi = 0, kmin = INT64_MAX, kmax = INT64_MIN;
  const uint64_t *base = stage + (size_t)s * FLUSH_Q * 32;
  static_assert(NS == 2 || NS == 4, "reduce_staged: lane j owns slot j % NS");
#pragma unroll
  for (int i = 0; i < NS; i++) {  // NS source lanes per lane group, rotated by the slot: conflict-free
    const uint32_t src = g * NS + ((i + s) & (NS - 1));
    const uint64_t c = base[src], v = base[32 + src];
    cnt += c;
    if (is_f64) {
      sum = (uint64_t)__double_as_longlong(__longlong_as_double((long long)sum) + __longlong_as_double((long long)v));
    } else {
      sum += v;
      if (VK != VK_GOR) hi += (int64_t)base[64 + src] + (sum < v ? 1 : 0);
    }
    const int64_t a = (int64_t)base[96 + src], b = (int64_t)base[128 + src];
    kmin = a < kmin ? a : kmin;
    kmax = b > kmax ? b : kmax;
  }
#pragma unroll
  for (int o = NS; o < 32; o <<= 1) {  // lanes j, j ^ o own the same slot
    cnt += shfl_xor_u64(cnt, o);
    const uint64_t v = shfl_xor_u64(sum, o);
    // (every shuffle outside the is_f64 branch: slots of a generic-kind warp can hold columns of different types)
    const int64_t vh = VK != VK_GOR ? (int64_t)shfl_xor_u64((uint64_t)hi, o) : 0;
    if (is_f64) {
      sum = (uint64_t)__double_as_longlong(__longlong_as_double((long long)sum) + __longlong_as_double((long long)v));
    } else {
      sum += v;
      if (VK != VK_GOR) hi += vh + (sum < v ? 1 : 0);
    }
    const int64_t a = (int64_t)shfl_xor_u64((uint64_t)kmin, o), b = (int64_t)shfl_xor_u64((uint64_t)kmax, o);
    kmin = a < kmin ? a : kmin;
    kmax = b > kmax ? b : kmax;
  }
  if (lane < n_slots && cnt)
    table_update(P, stab, cs, (uint64_t)(uint32_t)meta, cs.agg_mask, is_f64, (uint32_t)cnt, sum, hi, kmin, kmax);
  __syncwarp();
}

// Every lane parks its partial (identities unless `live`) in staging slot `seq`, the lane `meta_lane` records the slot's
// (query column << 32) | cell, and every NS slots the warp reduces them. Called by all 32 lanes.
template <int VK, int NS>
__device__ __forceinline__ void stage_partial(const ScanParams &P, uint64_t *stab, uint64_t *stage, uint32_t &seq, bool live,
                                              const ValueAcc<VK> &va, bool meta_lane, uint64_t gcell) {
  uint64_t *q = stage + (size_t)seq * FLUSH_Q * 32 + (threadIdx.x & 31);
  q[0] = live ? va.count : 0;
  q[32] = live ? va.sum : 0;  // 0 bits == +0.0
  if (VK != VK_GOR) q[64] = live ? (uint64_t)va.sum_hi : 0;
  q[96] = live ? (uint64_t)va.kmin : (uint64_t)INT64_MAX;
  q[128] = live ? (uint64_t)va.kmax : (uint64_t)INT64_MIN;
  if (meta_lane) stage[NS * FLUSH_Q * 32 + seq] = gcell;
  if (++seq == NS) {
    reduce_staged<VK, NS>(P, stab, stage, seq);
    seq = 0;
  }
}

// Flush of one finished run per flushing lane (no FIRST/LAST). `seq` = staged slots in use (warp-uniform).
template <int VK, int NS>
__device__ __forceinline__ void flush_runs(const ScanParams &P, uint64_t *stab, uint64_t *stage, uint32_t &seq, bool active,
                                           uint32_t qcol, uint64_t cell, uint8_t pt, uint8_t mask, const ValueAcc<VK> &va) {
  const uint32_t m = __ballot_sync(FULL, active);
  if (m == 0) return;
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t gcell = ((uint64_t)qcol << 32) | (uint32_t)cell;
  const int leader = __ffs(m) - 1;
  const uint64_t lcell = shfl_u64(gcell, leader);
  // (Not for GROUP BY series: its cells can exceed 32 bits, and its lanes never share one. GROUP BY tags keeps its cells
  // below 2^32, and its lanes share a cell whenever their series share a group.) The staged
  // path also serves tables too large for shared memory - the reduced partial then goes to the global state with one
  // atomic per quantity instead of 32 contended ones.
  const bool same = !P.group_by_series && __all_sync(FULL, !active || gcell == lcell);
  if (same) {
    stage_partial<VK, NS>(P, stab, stage, seq, active && va.count, va, (int)lane == leader, lcell);
  } else if (active && va.count) {  // lanes on different cells (GROUP BY series, unaligned pages): one update each
    table_update(P, stab, P.cols[qcol], cell, mask, VK == VK_GOR || (VK == VK_GEN && pt == TSKV_PT_F64), va.count, va.sum,
                 va.sum_hi, va.kmin, va.kmax);
  }
}

template <int K, typename S>
__device__ __forceinline__ bool cursor_exhausted(const DeltaCursor<K, S> &c) { return c.exhausted; }
template <bool ZZ>
__device__ __forceinline__ bool cursor_exhausted(const S8bCursor<ZZ> &c) { return c.exhausted(); }
template <int K, typename S>
__device__ __forceinline__ void cursor_reset(DeltaCursor<K, S> &c, uint32_t lane_ring) { c.bs.reset(lane_ring); }
template <bool ZZ>
__device__ __forceinline__ void cursor_reset(S8bCursor<ZZ> &c, uint32_t lane_ring) { c.reset(lane_ring); }

// Rows of an RLE time page that stay inside [t, t + d] when stepping by delta > 0 from t: min(left, floor(d / delta) + 1),
// with the quotient estimated in double precision (inv = 1.0 / delta, one division per page) and corrected exactly.
__device__ __forceinline__ uint32_t rle_rows_within(uint64_t d, uint64_t delta, double inv, uint32_t left) {
  const double e = (double)d * inv;
  if (e >= (double)left) return left;  // floor(d / delta) >= left - 1 (relative error 2^-51, left < 2^32)
  uint64_t q = (uint64_t)e;            // < 2^32, off by at most one
  if (__umul64hi(q, delta) != 0 || q * delta > d) q--;
  else if (d - q * delta >= delta) q++;
  return (uint32_t)min((uint64_t)left, q + 1);
}

// NARROW (simple8b integer values, no FIRST / LAST): every page of the chunk is narrow (ScanParams.page_narrow), so the
// values are decoded and accumulated in 32-bit arithmetic (S8bCursor::next32, ValueAcc::add32).
template <int TK, int VK, bool SEL, bool NARROW>
__device__ __forceinline__ void scan_chunk_seg(const ScanParams &P, uint32_t item_begin, uint32_t item_end,
                                               uint32_t ring_base, uint64_t *stab, uint64_t *stage, uint4 *s_tomb,
                                               uint32_t part, uint32_t n_parts, uint32_t part_rows) {
  constexpr int NS = flush_slots(TK);  // staging slots of the staged flush
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t item = item_begin + lane;
  const bool have_item = item < item_end;
  // this lane's slots in the warp's staging rings: [time ring (simple8b timestamps only)] [value ring]
  const uint32_t tslot = ring_base + lane * RING_BYTES;
  const uint32_t vslot = ring_base + (TK == TK_S8B ? RING_BYTES_PER_WARP : 0) + lane * RING_BYTES;

  uint32_t page = 0, slot = 0, qcol = 0, n_rows = 0;
  uint8_t pt = VK == VK_GOR ? TSKV_PT_F64 : TSKV_PT_I64, mask = 0;
  PageView tpv, vpv;
  S8bCursor<false> tcur;                       // TK_S8B: timestamps staged through the time ring
  uint64_t rle_t0 = 0, rle_delta = 0;          // TK_RLE: t(row) = rle_t0 + row * rle_delta (wrapping), closed form
  double rle_inv = 0.0;
  typename std::conditional<VK == VK_S8B, S8bCursor<true>, DeltaCursor<-1, SeqStream>>::type vcur_d;
  GorillaRing vcur_g;
  const uint32_t *vbm = nullptr;  // value validity bitmap, 32 rows per word
  const uint32_t *keepw = nullptr;  // row-filter keep bits of the column group (k_row_filter), or null
  bool allnull = false;
  int64_t pend_t = 0;  // timestamp of row `row`

  if (TK == TK_S8B) tcur.reset(tslot);
  if (VK == VK_GOR) vcur_g.reset(vslot);
  else cursor_reset(vcur_d, vslot);
  // This lane decodes rows [r0, n_rows) of its page: the whole page, or - the bin's pages are cut at restart points
  // (n_parts > 1, never with FIRST / LAST) - part `part` of it. A page without restart points (short, or its streams did
  // not decode cleanly when the index was built) is decoded whole by the lane of part 0, errors and all.
  uint32_t r0 = 0, page_rows = 0;
  if (have_item) {
    page = P.work_page[item];
    slot = P.work_slot[item];
    qcol = P.work_qcol[item] & 0x7f;
    const tskv_page_desc vd = P.descs[page];
    if (P.has_tomb) s_tomb[threadIdx.x] = tomb_lookup(P, vd.series_id, vd.column_id);
    const uint32_t tpage = P.time_page_of[page];
    const tskv_page_desc td = P.descs[tpage];
    if (VK != VK_GOR) pt = P.cols[qcol].phys_type;
    mask = P.cols[qcol].agg_mask;
    page_rows = vd.num_values;
    uint32_t sk_v = SKIP_NONE, sk_t = SKIP_NONE;  // the page's restart points (value stream, time stream)
    bool split = false;
    if (n_parts > 1 && page_rows > part_rows) {
      sk_v = __ldg(P.skip_off + page);
      sk_t = TK == TK_S8B ? __ldg(P.skip_off + tpage) : 0u;
      split = sk_v != SKIP_NONE && sk_t != SKIP_NONE;
    }
    r0 = part * part_rows;
    tskv_status st = kind_status(vd.reserved);  // the time page is RLE / simple8b here: always decodable
    if (part != 0 && (!split || r0 >= page_rows)) {
      // nothing for this lane: the page ends before this part, or part 0's lane decodes all of it
    } else if (st != TSKV_OK) {
      report_error(P, st, page);
    } else {
      tpv.open(P.arena, td);
      vpv.open(P.arena, vd);
      n_rows = split ? min(page_rows, r0 + part_rows) : page_rows;
      vbm = reinterpret_cast<const uint32_t *>(vpv.bitset);
      if (P.row_keep) keepw = P.row_keep + P.keep_off[tpage];
      const uint32_t ent = r0 / SKIP_ROWS - 1;  // restart point of row r0 (part != 0)
      if (TK == TK_RLE) {  // timestamp.rs:226-259
        DeltaCursor<DK_RLE_SC, BeStream> rc;
        st = rc.open(tpv, td.reserved);
        rle_delta = rc.delta;
        rle_t0 = rc.v + rc.delta;
        if ((int64_t)rle_delta > 0) rle_inv = 1.0 / (double)rle_delta;
      } else if (part == 0) {
        st = tcur.open(tpv, td.reserved, tslot);
      } else {
        tcur.restore(tpv, tslot, load_skip(P.skip + sk_t + ent));  // the state after row r0's timestamp
      }
      if (st == TSKV_OK) {
        if (part == 0) {
          if (VK == VK_GOR) vcur_g.open(vpv, vslot);
          else { st = vcur_d.open(vpv, vd.reserved, vslot); allnull = vd.reserved == DK_ALLNULL; }
        } else {
          const SkipEntry e = load_skip(P.skip + sk_v + ent);  // the state before the first value of row >= r0
          if constexpr (VK == VK_GOR) vcur_g.restore(vpv, vslot, e);
          else if constexpr (VK == VK_S8B) vcur_d.restore(vpv, vslot, e);
          // (generic value codecs are never cut: n_parts == 1)
        }
      }
      if (st == TSKV_OK && n_rows) {
        if (TK == TK_RLE) pend_t = (int64_t)(rle_t0 + (uint64_t)r0 * rle_delta);
        else if (part == 0) pend_t = (int64_t)tcur.next();  // the first value: no ring access (cursors.cuh)
        else pend_t = (int64_t)tcur.v;
      }
      if (st != TSKV_OK) { report_error(P, st, st == TSKV_ERR_BITSET_MISMATCH ? tpage : page); n_rows = 0; }
    }
  }
  const bool to_page_end = n_rows == page_rows;  // this lane reaches the end of the page's streams
  ring_drain();  // the rings' initial fills have landed before the first step (once per page)

  static_assert(!NARROW || (VK == VK_S8B && !SEL), "narrow chunks: simple8b integer values, no FIRST / LAST");
  ValueAcc<VK> va;
  va.reset(NARROW);
  RunAcc acc;  // flush image (+ first/last state when SEL)
  acc.first_ts = acc.last_ts = 0; acc.first_val = acc.last_val = 0; acc.first_ok = acc.last_ok = false;
  BucketState bk; bk.valid = false; bk.floor_regime = false; bk.lo = 0; bk.hi = 0; bk.idx = 0;
  bool have_run = false;
  uint32_t run_idx = 0;
  uint32_t row = r0;  // (a multiple of 32)
  if (n_rows == 0) row = 0;
  uint32_t n_points = 0, n_inrange = 0;
  uint32_t vword = 0, vahead = vbm ? __ldg(vbm + (row >> 5)) : 0;  // bitmap word of `row`, and the next one (prefetched)
  uint32_t kword = 0xffffffffu;                        // row-filter bits of the same 32 rows (all ones without predicates)
  bool first_pending = false;                          // FIRST/LAST: the run has not seen a kept row yet
  const uint64_t flip = pt == TSKV_PT_U64 ? 0x8000000000000000ull : 0ull;
  // (the FIRST / LAST variants read the slot and its group again at each flush: holding them takes registers those
  // kernels do not have, ptxas spills)
  const uint64_t group_base = SEL ? 0 : group_cell_base(P, slot);
  uint32_t staged = 0;  // staged flush slots in use (warp-uniform)

  // Finished runs of the flushing lanes -> partial tables.
  auto flush_now = [&](bool flush) {
    if (flush) va.fold(pt, NARROW);
    if (SEL) {
      if (__any_sync(FULL, flush)) {
        acc.count = va.count; acc.sum = va.sum; acc.sum_hi = va.sum_hi; acc.kmin = va.kmin; acc.kmax = va.kmax;
        const uint32_t fslot = have_item ? __ldg(P.work_slot + item) : 0u;
        warp_flush<SEL>(P, stab, flush, qcol, group_cell_base(P, fslot) + run_idx, (int64_t)run_idx, pt, mask, acc, fslot);
      }
    } else {
      flush_runs<VK, NS>(P, stab, stage, staged, flush, qcol, group_base + run_idx, pt, mask, va);
    }
  };
  // One row's value: validity bit, decode (every valid row is decoded - rows outside the time ranges too, the streams
  // are sequential), accumulate when the segment is selected. Returns the value; `vv` = the row holds one.
  auto row_value = [&](bool accumulate, bool &vv, bool &kept) -> uint64_t {
    if ((row & 31) == 0) {  // entering a new bitmap word: take the prefetched one, prefetch the next
      vword = vahead;
      vahead = __ldg(vbm + (row >> 5) + 1);  // reads at most 8 bytes past the bitmap (inside the page)
      if (keepw) kword = __ldg(keepw + (row >> 5));
    }
    vv = ((vword >> (row & 31)) & 1) && !allnull;
    kept = (kword >> (row & 31)) & 1;
    uint64_t v = 0;
    if (vv) {
      n_points++;
      if constexpr (NARROW) {
        const uint32_t v32 = vcur_d.next32();
        if (accumulate && kept) { va.count++; va.add32(v32); }
      } else {
        v = VK == VK_GOR ? vcur_g.next() : vcur_d.next();
        if (accumulate && kept) { va.count++; va.add(v, pt, flip); }
      }
    }
    return v;  // (0 for narrow chunks: only FIRST / LAST use it)
  };
  // The next value, accumulated when `take` (every value is decoded: the streams are sequential).
  auto next_add = [&](bool take) {
    if constexpr (NARROW) {
      const uint32_t v32 = vcur_d.next32();
      if (take) va.add32(v32);
    } else {
      const uint64_t v = VK == VK_GOR ? vcur_g.next() : vcur_d.next();
      if (take) va.add(v, pt, flip);
    }
  };
  auto check_values = [&]() {
    const bool bad = VK == VK_GOR ? vcur_g.failed() : cursor_exhausted(vcur_d);
    if (bad) {
      report_error(P, (VK == VK_GOR && vcur_g.overran()) ? TSKV_ERR_SHORT_BLOCK : TSKV_ERR_BITSET_MISMATCH, page);
      n_rows = 0;
      have_run = false;
    }
  };

  // ---- RLE timestamps, increasing, at most one time range, no tombstones: the segment structure is arithmetic in the
  // ROW index. Rows [ra, rb1) are inside the range; bucket edges advance by q or q + 1 rows (w = q * delta + rem, the
  // offset e of a bucket's first row inside it decides), so a segment costs a handful of 32-bit operations instead of
  // 64-bit interval arithmetic per segment. Anything else (wrapping / constant timestamps, several ranges, tombstones,
  // the reference's truncating-% regime for negative dividends, values near the i64 limits) takes the general logic.
  uint32_t ra = 0, rb1 = 0, nb = 0xffffffffu, q32 = 0, bidx = 0;
  uint64_t e_off = 0, w_rem = 0;
  bool fast = false;
  if (TK == TK_RLE) {
    bool elig = P.n_ranges <= 1 && !P.has_tomb;
    if (elig && n_rows) {
      // (the parts of a page may take different paths: both give the same result)
      const uint64_t span_t = (uint64_t)(page_rows - 1) * rle_delta;
      elig = (int64_t)rle_delta > 0 && __umul64hi((uint64_t)(page_rows - 1), rle_delta) == 0 && span_t < (1ull << 62) &&
             rle_t0 + (1ull << 62) < (1ull << 63) && rle_t0 + span_t + (1ull << 62) < (1ull << 63) &&
             P.width < ((int64_t)1 << 61);  // (every row < 2^62 and |origin_mod| < 2^61: no dividend t - origin_mod + width wraps)
      if (elig) {
        const int64_t t0 = (int64_t)rle_t0;
        ra = 0;
        rb1 = page_rows;
        if (P.n_ranges == 1) {  // rows with t < a, rows with t <= b
          const int64_t a = P.ranges[0].min_ts, b = P.ranges[0].max_ts;
          ra = a <= t0 ? 0u : rle_rows_within((uint64_t)(a - 1) - rle_t0, rle_delta, rle_inv, page_rows);
          rb1 = b < t0 ? 0u : rle_rows_within((uint64_t)b - rle_t0, rle_delta, rle_inv, page_rows);
        }
        ra = min(max(ra, row), n_rows);  // this lane's rows: [row, n_rows)
        rb1 = min(max(rb1, row), n_rows);
        if (P.width > 0 && ra < rb1) {
          const int64_t tr = (int64_t)(rle_t0 + (uint64_t)ra * rle_delta);
          if ((int64_t)((uint64_t)tr - (uint64_t)P.origin_mod + (uint64_t)P.width) < 0) {
            elig = false;  // truncating-% regime (time_window.rs:184-198): general logic
          } else if (!locate_bucket(P, tr, bk)) {
            report_error(P, TSKV_ERR_BUCKET_RANGE, page);
            n_rows = 0;
          } else {
            bidx = bk.idx;
            nb = rle_rows_within((uint64_t)bk.hi - (uint64_t)tr, rle_delta, rle_inv, 0xffffffffu);
            e_off = (uint64_t)tr + (uint64_t)nb * rle_delta - ((uint64_t)bk.hi + 1);
            q32 = rle_rows_within((uint64_t)P.width, rle_delta, rle_inv, 0xffffffffu) - 1;
            w_rem = (uint64_t)P.width - (uint64_t)q32 * rle_delta;
          }
        }
      }
    }
    fast = __all_sync(FULL, elig);
  }

  // ---- Uniform schedule (RLE timestamps, GROUP BY bucket or tags, no FIRST / LAST). When every lane that holds rows starts at
  // the same row and time, steps by the same delta, has the same range rows [ra, rb1), the same bucket state and the same
  // query column (TSBS-aligned pages: 80 % of C4's), the bucket edges fall on the same rows in every lane. The warp then
  // walks ONE schedule, the leader's: per bitmap word one dense / sparse vote, per bucket its rows and one staged store
  // per lane - no per-lane segment state, no alignment reduction, no ballot / same-cell vote, since all lanes close the
  // same cell. The staged partials and their order are the ones the segment loop below makes for such a warp. Lanes
  // without rows walk along idle; a lane whose values run out stops decoding as there. (Not for the generic value
  // codecs: their larger cursor leaves no registers for a second loop.)
  if (TK == TK_RLE && VK != VK_GEN && !SEL && fast && P.width > 0 && !P.group_by_series) {
    const bool mine = row < n_rows;
    const uint32_t with_rows = __ballot_sync(FULL, mine);
    const int src = with_rows ? __ffs(with_rows) - 1 : 0;
    const uint64_t t_first = rle_t0 + (uint64_t)row * rle_delta;
    // (`&`, not `&&`: every lane must reach every shuffle. GROUP BY tags: the lanes' groups agree too, and a group's
    // cells stay below 2^32)
    const bool agree = (shfl_u64(rle_delta, src) == rle_delta) & (shfl_u64(t_first, src) == t_first) &
                       (shfl_u64(e_off, src) == e_off) & (__shfl_sync(FULL, row, src) == row) &
                       (__shfl_sync(FULL, n_rows, src) == n_rows) & (__shfl_sync(FULL, ra, src) == ra) &
                       (__shfl_sync(FULL, rb1, src) == rb1) & (__shfl_sync(FULL, bidx, src) == bidx) &
                       (__shfl_sync(FULL, nb, src) == nb) & (__shfl_sync(FULL, qcol, src) == qcol) &
                       (__shfl_sync(FULL, (uint32_t)group_base, src) == (uint32_t)group_base);
    if (with_rows && __all_sync(FULL, !mine || agree)) {
      // the leader's schedule in every lane (lanes without rows may hold other values)
      rle_delta = shfl_u64(rle_delta, src);
      e_off = shfl_u64(e_off, src);
      w_rem = shfl_u64(w_rem, src);
      q32 = __shfl_sync(FULL, q32, src);
      row = __shfl_sync(FULL, row, src);
      ra = __shfl_sync(FULL, ra, src);
      rb1 = __shfl_sync(FULL, rb1, src);
      bidx = __shfl_sync(FULL, bidx, src);
      nb = __shfl_sync(FULL, nb, src);
      const uint64_t col = ((uint64_t)__shfl_sync(FULL, qcol, src) << 32) | __shfl_sync(FULL, (uint32_t)group_base, src);
      uint32_t end = __shfl_sync(FULL, n_rows, src);
      while (row < end) {  // one bitmap word per pass (`row` is a multiple of 32 here)
        if (n_rows) {      // this lane still decodes: take the prefetched word, prefetch the next
          vword = vahead;
          vahead = __ldg(vbm + (row >> 5) + 1);  // reads at most 8 bytes past the bitmap (inside the page)
          if (keepw) kword = __ldg(keepw + (row >> 5));
        }
        const uint32_t wend = min(row + 32, end);
        const uint32_t m = (n_rows && !allnull) ? vword & (0xffffffffu >> (32 - (wend - row))) : 0u;  // rows holding a value
        const uint32_t lo = min(max(ra, row), wend) - row, hi = max(min(max(rb1, row), wend) - row, lo);
        const uint32_t take = m & kword & (uint32_t)((1ull << hi) - (1ull << lo));  // rows whose value is accumulated
        // Dense words (every row holding a value is kept, on all lanes) decode popc values with no test per row.
        // The vote only chooses the speed: both loops give the same result.
        const bool dense = __all_sync(FULL, take == m);
        uint32_t r = row;
        while (r < wend) {  // the word's pieces: rows before the range, one per bucket, rows after it
          const bool in = r >= ra && r < rb1;
          uint32_t pend = r < ra ? min(ra, wend) : wend;
          if (in) {
            if (nb == 0) {  // next bucket (one narrower than the step may hold no row at all)
              do {
                bidx++;
                nb = q32 + (e_off < w_rem ? 1u : 0u);
                e_off = e_off + (uint64_t)nb * rle_delta - (uint64_t)P.width;
              } while (nb == 0);
              if (bidx >= P.n_buckets) {
                if (n_rows) { report_error(P, TSKV_ERR_BUCKET_RANGE, page); n_rows = r; }
                end = r;
                break;
              }
            }
            const uint32_t lim = min(rb1, wend);
            pend = nb < lim - r ? r + nb : lim;
            nb -= pend - r;
          }
          const uint32_t pmask = (uint32_t)((1ull << (pend - row)) - (1ull << (r - row)));
          const uint32_t mp = n_rows ? m & pmask : 0u, tp = take & mp;
          n_points += __popc(mp);
          if (in && n_rows) n_inrange += __popc(kword & pmask);
          va.count += __popc(tp);
          if (dense) {
#pragma unroll 1
            for (uint32_t n = __popc(mp); n; n--) next_add(true);
          } else {  // only the rows holding a value
#pragma unroll 1
            for (uint32_t b = mp; b; b &= b - 1) next_add(tp & b & (0u - b));
          }
          r = pend;
          if (n_rows) check_values();
          if (in && (nb == 0 || r == rb1)) {  // the bucket's last row: its partial goes to the staging area
            va.fold(pt, NARROW);
            stage_partial<VK, NS>(P, stab, stage, staged, n_rows && va.count, va, lane == 0, col + bidx);
            va.reset(NARROW);
          }
        }
        row = r;
      }
      row = n_rows;  // nothing is left for the segment loop below
    }
  }

  // The warp walks its 32 pages SEGMENT by segment (a segment = rows of one page sharing (selected, bucket)), and for
  // GROUP BY bucket / tags it keeps the lanes aligned on the BUCKET: in every iteration only the lanes whose next selected
  // segment lies in the smallest pending bucket go ahead (the others keep their segment pending, at most an iteration
  // or two). Pages whose first row falls just before a bucket edge would otherwise run one segment ahead of their
  // neighbours for the whole page, no two lanes would ever finish a run for the same cell in the same iteration, and
  // every flush would degenerate into 32 contended atomics instead of one staged store per lane.
  const bool align = P.width > 0 && !P.group_by_series;
  bool pending = false;
  uint32_t seg_n = 0, seg_b = 0;  // pending segment: rows (RLE pages), bucket
  bool seg_in = false, seg_masked = false;
  int64_t lim_lo = 0, lim_hi = 0;  // pending segment (simple8b timestamps): closed interval its rows stay in
  for (;;) {
    const bool has = row < n_rows;
    if (!__any_sync(FULL, has || have_run)) break;
    // ---- 1. attributes of the next segment ------------------------------------------------------------
    if (has && !pending) {
      pending = true;
      seg_in = false;
      seg_masked = false;
      seg_n = 0;
      if (TK == TK_RLE && fast) {
        if (row < ra) seg_n = ra - row;
        else if (row >= rb1) seg_n = n_rows - row;
        else {
          seg_in = true;
          while (nb == 0) {  // next bucket (one narrower than the step may hold no row at all)
            bidx++;
            nb = q32 + (e_off < w_rem ? 1u : 0u);
            e_off = e_off + (uint64_t)nb * rle_delta - (uint64_t)P.width;
          }
          if (bidx >= P.n_buckets) {
            report_error(P, TSKV_ERR_BUCKET_RANGE, page);
            seg_in = false;
            n_rows = row;
            pending = false;
          } else {
            seg_n = min(nb, rb1 - row);
            seg_b = bidx;
            if (P.width > 0) nb -= seg_n;
          }
        }
      } else {
        lim_lo = lim_hi = pend_t;
        seg_in = range_span(P, pend_t, lim_lo, lim_hi);
        if (P.has_tomb) {  // decode_pages' tombstone handling (reader.rs:507-551) as two more segment attributes
          const uint4 tl = s_tomb[threadIdx.x];
          const bool dropped = tomb_span(P.tomb_ranges, P.n_tomb_global, pend_t, lim_lo, lim_hi) |
                               tomb_span(P.tomb_ranges + tl.x, tl.y, pend_t, lim_lo, lim_hi);
          seg_masked = tomb_span(P.tomb_ranges + tl.z, tl.w, pend_t, lim_lo, lim_hi);
          if (dropped) seg_in = false;
        }
        if (seg_in) {
          if (!(bk.valid && pend_t >= bk.lo && pend_t <= bk.hi) && !locate_bucket(P, pend_t, bk)) {
            report_error(P, TSKV_ERR_BUCKET_RANGE, page);
            seg_in = false;
            bk.valid = false;
            lim_lo = lim_hi = pend_t;
          } else {
            lim_lo = lim_lo > bk.lo ? lim_lo : bk.lo;
            lim_hi = lim_hi < bk.hi ? lim_hi : bk.hi;
            seg_b = bk.idx;
          }
        }
        if (TK == TK_RLE) {  // the segment's row count: closed form, or a walk for constant / wrapping timestamps
          const uint32_t left = n_rows - row;
          if ((int64_t)rle_delta > 0) {
            seg_n = rle_rows_within((uint64_t)lim_hi - (uint64_t)pend_t, rle_delta, rle_inv, left);
          } else {
            int64_t t = pend_t;
            do {
              seg_n++;
              t = (int64_t)((uint64_t)t + rle_delta);
            } while (seg_n < left && t >= lim_lo && t <= lim_hi);
          }
        }
      }
    }
    // ---- 2. bucket alignment, run bookkeeping, flush ------------------------------------------------------
    bool go = pending;
    if (align) {
      const uint32_t bmin = __reduce_min_sync(FULL, (pending && seg_in) ? seg_b : 0xffffffffu);
      go = pending && (!seg_in || seg_b == bmin);
    }
    const bool newrun = go && seg_in && (!have_run || seg_b != run_idx);
    const bool flush = have_run && (newrun || !has);
    flush_now(flush);
    if (flush) have_run = false;
    if (newrun) {
      have_run = true;
      run_idx = seg_b;
      va.reset(NARROW);
      if (SEL) { acc.first_ok = acc.last_ok = false; first_pending = true; }
    }
    // ---- 3. the segment's rows --------------------------------------------------------------------------
    if (go) {
      pending = false;
      const bool accumulate = seg_in && !seg_masked;
      if (TK == TK_RLE) {
        // the row count is known: values one bitmap word at a time (no per-row timestamp, no per-row bitmap fetch)
        const uint32_t rend = row + seg_n;
        uint32_t r = row;
        while (r < rend) {
          if ((r & 31) == 0) {  // entering a new bitmap word: take the prefetched one, prefetch the next
            vword = vahead;
            vahead = __ldg(vbm + (r >> 5) + 1);  // reads at most 8 bytes past the bitmap (inside the page)
            if (keepw) kword = __ldg(keepw + (r >> 5));
          }
          const uint32_t off = r & 31;
          const uint32_t span = min(32u - off, rend - r);
          const uint32_t smask = 0xffffffffu >> (32 - span);
          const uint32_t m = allnull ? 0u : ((vword >> off) & smask);  // rows holding a value
          const uint32_t kb = (kword >> off) & smask;                   // rows the row filter keeps
          n_points += __popc(m);
          if (seg_in) n_inrange += __popc(kb);
          if (!SEL) {
            const uint32_t take = accumulate ? (m & kb) : 0u;  // rows whose value is accumulated
            va.count += __popc(take);
            // Dense spans (every row holds a value and is kept: every span of a page without nulls when the query has no
            // field predicates - C4 generates 5 % nulls on 1 % of its pages, bench.py) decode popc(m) values with no test
            // per row. The lanes choose together: a lane on the other loop would run it after them. (Both loops give the
            // same result, so which lanes the vote sees only decides the speed.)
            if (__all_sync(__activemask(), take == m)) {
#pragma unroll 1
              for (uint32_t n = __popc(m); n; n--) next_add(true);
            } else {  // only the rows holding a value
#pragma unroll 1
              for (uint32_t b = m; b; b &= b - 1) next_add(take & b & (0u - b));
            }
          } else {  // FIRST / LAST wanted: the run's first and last KEPT rows keep (ts, value, valid)
            for (uint32_t j = 0; j < span; j++) {
              bool vv = (m >> j) & 1;
              uint64_t v = 0;
              if (vv) v = VK == VK_GOR ? vcur_g.next() : vcur_d.next();
              vv = vv && !seg_masked;
              if (seg_in && ((kb >> j) & 1)) {
                const int64_t t = (int64_t)(rle_t0 + (uint64_t)(r + j) * rle_delta);
                if (first_pending) { acc.first_ts = t; acc.first_val = vv ? v : 0; acc.first_ok = vv; first_pending = false; }
                acc.last_ts = t;
                acc.last_val = vv ? v : 0;
                acc.last_ok = vv;
                if (vv) { va.count++; va.add(v, pt, flip); }
              }
            }
          }
          r += span;
        }
        row = rend;
        if (!(TK == TK_RLE && fast)) pend_t = (int64_t)(rle_t0 + (uint64_t)rend * rle_delta);
      } else {
        // simple8b timestamps: ONE loop decodes the row's value and the NEXT row's timestamp - two independent dependent
        // chains in flight per lane - and stops at the first timestamp outside the segment's interval
        int64_t t = pend_t;
        const uint64_t span = (uint64_t)lim_hi - (uint64_t)lim_lo;
        bool more;
#pragma unroll 1
        do {
          bool vv, kept;
          const uint64_t v = row_value(accumulate, vv, kept);
          if (SEL && seg_in && kept) {
            const bool ok = vv && !seg_masked;
            if (first_pending) { acc.first_ts = t; acc.first_val = ok ? v : 0; acc.first_ok = ok; first_pending = false; }
            acc.last_ts = t;
            acc.last_val = ok ? v : 0;
            acc.last_ok = ok;
          }
          if (seg_in && kept) n_inrange++;
          row++;
          t = (int64_t)tcur.next();  // (past the last row this runs one value too far - harmless)
          more = row < n_rows && (uint64_t)t - (uint64_t)lim_lo <= span;
        } while (more);
        pend_t = t;
        if (tcur.exhausted() && row < n_rows) { report_error(P, TSKV_ERR_BITSET_MISMATCH, P.time_page_of[page]); n_rows = row; }
      }
      check_values();
    }
  }
  if (!SEL && staged) {  // partials still parked in the staging area
    reduce_staged<VK, NS>(P, stab, stage, staged);
    staged = 0;
  }
  // (only the lane that decodes the page's last rows walks on to the sentinel)
  if (VK == VK_GOR && have_item && n_rows != 0 && to_page_end && vcur_g.consumed_any() && !vcur_g.drain())  // float.rs:480-591
    report_error(P, TSKV_ERR_SHORT_BLOCK, page);
  ring_drain();  // nothing in flight when the next chunk reuses the rings
  n_points = __reduce_add_sync(FULL, n_points);
  n_inrange = __reduce_add_sync(FULL, n_inrange);
  if (lane == 0) {
    if (n_points) atomicAdd(&P.stats[0], (unsigned long long)n_points);
    if (n_inrange) atomicAdd(&P.stats[1], (unsigned long long)n_inrange);
  }
}

// The fused decode -> filter -> bucket-reduce kernel, one instantiation per decode-kind bin (time codec x
// value codec) and SEL (= the query asks for FIRST/LAST) so that each keeps its state in registers.
// The bins' kernels run concurrently on separate streams, each with a persistent grid sized to its share
// of the work; a warp repeatedly grabs one 32-item chunk of its bin from the bin's global counter.
#ifndef SCAN_MIN_BLOCKS
#define SCAN_MIN_BLOCKS 4
#endif
// 4 blocks of 4 warps per SM: 128 registers per thread. On sm_90a (ptxas -v) that keeps the variants without FIRST /
// LAST free of spills; the FIRST / LAST variants spill 4-146 bytes. A fifth block per SM would cap them at 96 registers
// and move the row loop's state into local memory.
__host__ __device__ constexpr int scan_min_blocks(int /*tk*/, bool /*sel*/) { return SCAN_MIN_BLOCKS; }
// staging-ring bytes one warp of the fused kernel needs (generic time pages read from global memory)
__host__ __device__ constexpr uint32_t scan_ring_bytes_per_warp(int tk) {
  return tk == TK_RLE ? RING_BYTES_PER_WARP : tk == TK_S8B ? 2 * RING_BYTES_PER_WARP : 0;
}
// per-warp shared memory of the fused kernel: staging rings + the staged-flush area
__host__ __device__ constexpr uint32_t scan_warp_bytes(int tk) {
  return tk == TK_GEN ? 0 : scan_ring_bytes_per_warp(tk) + flush_stage_bytes(flush_slots(tk));
}
// per-lane tombstone lists (tomb_lookup), after the warps' areas; allocated only when the page set has tombstones
constexpr uint32_t SCAN_TOMB_BYTES = SCAN_THREADS * sizeof(uint4);
// Narrow pages of a simple8b-value bin (ScanParams.page_narrow), per page set: none, some or all of them. NARROW_SOME
// kernels choose per chunk; NARROW_ALL kernels hold the narrow arithmetic only (a kernel that holds both row loops runs
// its narrow chunks ~1.5 % slower on C4: H100, see DESIGN.md §5).
enum { NARROW_NONE = 0, NARROW_SOME = 1, NARROW_ALL = 2 };
template <int TK, int VK, bool SEL, int NARROW>
__global__ void __launch_bounds__(SCAN_THREADS, scan_min_blocks(TK, SEL)) k_scan_aggregate(const __grid_constant__ ScanParams P, int bin) {
  static_assert(NARROW == NARROW_NONE || (TK != TK_GEN && VK == VK_S8B && !SEL), "narrow kernels: simple8b values, no FIRST / LAST");
  // dynamic shared memory: [per-CTA partial table, P.smem_words 8-byte words (or empty)] [per warp: a value ring,
  // preceded by a time ring when the timestamps are simple8b, then the staged-flush area] [tombstone lists, only when
  // P.has_tomb]
  extern __shared__ __align__(16) uint64_t s_tab[];
  if (P.use_smem) {  // identities: 0 for counts / sums, +-inf keys for min / max
    for (uint32_t i = threadIdx.x; i < P.smem_words; i += SCAN_THREADS) s_tab[i] = 0;
    __syncthreads();
    for (uint32_t c = 0; c < P.n_cols; c++) {
      const ColState cs = P.cols[c];
      for (uint32_t i = threadIdx.x; i < (uint32_t)P.n_cells; i += SCAN_THREADS) {
        if (cs.agg_mask & TSKV_AGG_MIN) s_tab[cs.s_min + i] = 0x7fffffffffffffffull;
        if (cs.agg_mask & TSKV_AGG_MAX) s_tab[cs.s_max + i] = 0x8000000000000000ull;
      }
    }
    __syncthreads();
  }
  const uint32_t lane = threadIdx.x & 31;
  uint64_t *warp_area = s_tab + ((P.smem_words + 1) & ~1u) + (size_t)(threadIdx.x >> 5) * (scan_warp_bytes(TK) / 8);
  const uint32_t ring_base = (uint32_t)__cvta_generic_to_shared(warp_area);
  uint64_t *stage = warp_area + scan_ring_bytes_per_warp(TK) / 8;
  uint4 *s_tomb = reinterpret_cast<uint4 *>(s_tab + ((P.smem_words + 1) & ~1u) + (SCAN_THREADS / 32) * (scan_warp_bytes(TK) / 8));
  const uint32_t begin0 = __ldg(P.bin_cstart + bin), end0 = __ldg(P.bin_cstart + bin + 1);
  // pages cut at restart points: n_parts chunks per group of 32 pages (consecutive chunk numbers = the parts of one group)
  const uint32_t n_parts = (TK == TK_GEN || VK == VK_GEN || SEL) ? 1u : P.bin_parts[bin];
  const uint32_t part_rows = P.bin_part_rows[bin];
  const uint32_t n_chunks = ((end0 - begin0 + 31) >> 5) * n_parts;
  for (;;) {
    uint32_t c = 0;
    if (lane == 0) c = atomicAdd(P.task_counter + bin, 1u);
    c = __shfl_sync(FULL, c, 0);
    if (c >= n_chunks) break;
    const uint32_t group = n_parts > 1 ? c / n_parts : c;
    const uint32_t part = c - group * n_parts;
    const uint32_t begin = begin0 + (group << 5);
    const uint32_t end = min(begin + 32, end0);
    if constexpr (TK == TK_GEN) {
      scan_chunk_rows<TK, VK, SEL>(P, begin, end, ring_base, s_tab, s_tomb);
    } else if constexpr (NARROW == NARROW_SOME) {
      // 32-bit arithmetic when all of the chunk's pages are narrow (the work list keeps a bin's narrow pages together)
      const uint32_t item = begin + lane;
      const bool narrow = __all_sync(FULL, item >= end || __ldg(P.page_narrow + __ldg(P.work_page + item)));
      if (narrow) scan_chunk_seg<TK, VK, SEL, true>(P, begin, end, ring_base, s_tab, stage, s_tomb, part, n_parts, part_rows);
      else scan_chunk_seg<TK, VK, SEL, false>(P, begin, end, ring_base, s_tab, stage, s_tomb, part, n_parts, part_rows);
    } else {
      scan_chunk_seg<TK, VK, SEL, NARROW == NARROW_ALL>(P, begin, end, ring_base, s_tab, stage, s_tomb, part, n_parts, part_rows);
    }
  }
  if (P.use_smem) {  // merge this CTA's table into the global state, once
    __syncthreads();
    for (uint32_t c = 0; c < P.n_cols; c++) {
      const ColState cs = P.cols[c];
      const bool f64 = cs.phys_type == TSKV_PT_F64;
      for (uint32_t i = threadIdx.x; i < (uint32_t)P.n_cells; i += SCAN_THREADS) {
        const uint64_t cnt = s_tab[cs.s_count + i];
        if (!cnt) continue;
        atomicAdd(reinterpret_cast<unsigned long long *>(P.state + cs.count_off + i), (unsigned long long)cnt);
        if (cs.agg_mask & (TSKV_AGG_SUM | TSKV_AGG_MEAN)) {
          const uint64_t sv = s_tab[cs.s_sum + i];
          if (f64) atomicAdd(reinterpret_cast<double *>(P.state + cs.sum_off + i), __longlong_as_double((long long)sv));
          else add_int_sum(P.state + cs.sum_off + i, P.state + cs.sumhi_off + i, cs.agg_mask, sv,
                           (cs.agg_mask & TSKV_AGG_MEAN) ? (int64_t)s_tab[cs.s_hi + i] : 0);
        }
        if (cs.agg_mask & TSKV_AGG_MIN) atomicMin(reinterpret_cast<long long *>(P.state + cs.min_off + i), (long long)s_tab[cs.s_min + i]);
        if (cs.agg_mask & TSKV_AGG_MAX) atomicMax(reinterpret_cast<long long *>(P.state + cs.max_off + i), (long long)s_tab[cs.s_max + i]);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// state init / export / finalize
// ------------------------------------------------------------------------------------------------
struct StateLayout {
  uint64_t sum_i64_off, sum_i64_len;  // counts + integer sums
  uint64_t sum_f64_off, sum_f64_len;
  uint64_t min_off, min_len;          // MIN keys then exported FIRST keys
  uint64_t max_off, max_len;          // MAX keys then exported LAST keys
  uint64_t selval_off, selval_len;    // exported FIRST values then LAST values
  uint64_t first_pairs_off, first_cells;  // {key,val} pairs used by the scan kernel
  uint64_t last_pairs_off, last_cells;
  uint64_t first_keys_off, last_keys_off; // inside the min / max sections
  uint64_t snap_off;                      // snapshot of local first+last keys (multi-GPU masking)
  uint64_t total;
};

// Identities of the partial state; the same launch zeroes the scan's small per-pass scratch (task counters / status /
// counters, bin starts, work-list buckets) so that a pass starts with ONE node instead of three memsets + a kernel.
__global__ void k_init_state(uint64_t *state, StateLayout L, unsigned long long *aux, uint32_t aux_words, uint32_t *zero32,
                             uint32_t n_zero32, uint32_t *zero32b, uint32_t n_zero32b) {
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t k = i; k < aux_words; k += stride) aux[k] = 0;
  for (uint64_t k = i; k < n_zero32; k += stride) zero32[k] = 0;
  for (uint64_t k = i; k < n_zero32b; k += stride) zero32b[k] = 0;
  for (uint64_t k = i; k < L.total; k += stride) {
    uint64_t v = 0;
    if (k >= L.min_off && k < L.min_off + L.min_len) v = 0x7fffffffffffffffull;
    else if (k >= L.max_off && k < L.max_off + L.max_len) v = 0x8000000000000000ull;
    else if (k >= L.first_pairs_off && k < L.first_pairs_off + 2 * L.first_cells) v = ((k - L.first_pairs_off) & 1) ? 0 : 0x7fffffffffffffffull;
    else if (k >= L.last_pairs_off && k < L.last_pairs_off + 2 * L.last_cells) v = ((k - L.last_pairs_off) & 1) ? 0 : 0x8000000000000000ull;
    state[k] = v;
  }
}

// MEAN on an integer column: (hi:lo) exact sum -> f64 cell of the SUM_F64 section.
struct MeanExport {
  uint64_t lo_off, hi_off, dst_off;
  uint32_t is_signed, pad;
};

// De-interleave the {key,val} pairs into the contiguous key / value sections and convert the exact
// integer sums of MEAN columns to f64.
__global__ void k_export_pairs(uint64_t *state, StateLayout L, const MeanExport *means, uint32_t n_means,
                               uint64_t n_cells) {
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint32_t m = 0; m < n_means; m++) {
    const MeanExport me = means[m];
    for (uint64_t k = i; k < n_cells; k += stride) {
      uint64_t lo = state[me.lo_off + k];
      int64_t hi = (int64_t)state[me.hi_off + k];
      double d;
      if (me.is_signed) d = (double)(((__int128)hi << 64) + (__int128)(unsigned __int128)lo);
      else d = (double)(((unsigned __int128)(uint64_t)hi << 64) | (unsigned __int128)lo);
      state[me.dst_off + k] = (uint64_t)__double_as_longlong(d);
    }
  }
  for (uint64_t k = i; k < L.first_cells; k += stride) {
    state[L.first_keys_off + k] = state[L.first_pairs_off + 2 * k];
    state[L.selval_off + k] = state[L.first_pairs_off + 2 * k + 1];
  }
  for (uint64_t k = i; k < L.last_cells; k += stride) {
    state[L.last_keys_off + k] = state[L.last_pairs_off + 2 * k];
    state[L.selval_off + L.first_cells + k] = state[L.last_pairs_off + 2 * k + 1];
  }
}

// Sliding windows (tskvgpu_scan_prepare_sliding): the fused kernels aggregate into panes one slide wide; window j of a
// group is the fold of its panes j - k + 1 .. j (those that exist: pane p starts k - 1 slides after window p). One op
// per state array of the window layout that the kernels fill (counts, sums, min / max keys).
enum { COMBINE_ADD = 0, COMBINE_INT_SUM = 1, COMBINE_F64_SUM = 2, COMBINE_MIN = 3, COMBINE_MAX = 4 };
struct CombineOp {
  uint64_t pane_off, win_off;        // the array in the pane state / in the window state
  uint64_t pane_hi_off, win_hi_off;  // COMBINE_INT_SUM with has_hi: high words of the exact 128-bit sum (MEAN)
  uint32_t kind, has_hi;
};

// One thread per (op = blockIdx.y, group, window). Counts and integer sums add (wrapping low word; with has_hi the
// carries go to the high word), f64 sums add in pane order, min / max keys take the min / max.
__global__ void k_window_combine(const uint64_t *pane, uint64_t *win, const CombineOp *ops, uint32_t n_groups,
                                 uint32_t n_windows, uint32_t n_panes, uint32_t k) {
  const CombineOp op = ops[blockIdx.y];
  const uint64_t n = (uint64_t)n_groups * n_windows;
  for (uint64_t c = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; c < n; c += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t g = c / n_windows;
    const uint32_t j = (uint32_t)(c - g * n_windows);
    const uint32_t p0 = j + 1 >= k ? j + 1 - k : 0, p1 = j < n_panes - 1 ? j : n_panes - 1;
    const uint64_t *src = pane + op.pane_off + g * n_panes;
    switch (op.kind) {
      case COMBINE_INT_SUM: {
        const uint64_t *src_hi = pane + op.pane_hi_off + g * n_panes;
        uint64_t lo = 0, hi = 0;
        for (uint32_t p = p0; p <= p1; p++) {
          const uint64_t v = src[p];
          lo += v;
          hi += (lo < v ? 1u : 0u) + (op.has_hi ? src_hi[p] : 0u);
        }
        win[op.win_off + c] = lo;
        if (op.has_hi) win[op.win_hi_off + c] = hi;
        break;
      }
      case COMBINE_F64_SUM: {
        double acc = 0.0;
        for (uint32_t p = p0; p <= p1; p++) acc += __longlong_as_double((long long)src[p]);
        win[op.win_off + c] = (uint64_t)__double_as_longlong(acc);
        break;
      }
      case COMBINE_MIN: {
        int64_t acc = INT64_MAX;
        for (uint32_t p = p0; p <= p1; p++) acc = (int64_t)src[p] < acc ? (int64_t)src[p] : acc;
        win[op.win_off + c] = (uint64_t)acc;
        break;
      }
      case COMBINE_MAX: {
        int64_t acc = INT64_MIN;
        for (uint32_t p = p0; p <= p1; p++) acc = (int64_t)src[p] > acc ? (int64_t)src[p] : acc;
        win[op.win_off + c] = (uint64_t)acc;
        break;
      }
      default: {
        uint64_t acc = 0;
        for (uint32_t p = p0; p <= p1; p++) acc += src[p];
        win[op.win_off + c] = acc;
      }
    }
  }
}

__global__ void k_snapshot_keys(uint64_t *state, StateLayout L) {
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t k = i; k < L.first_cells; k += stride) state[L.snap_off + k] = state[L.first_keys_off + k];
  for (uint64_t k = i; k < L.last_cells; k += stride) state[L.snap_off + L.first_cells + k] = state[L.last_keys_off + k];
}

// After the key all-reduce: ranks whose local key lost contribute 0 to the value SUM all-reduce.
__global__ void k_mask_values(uint64_t *state, StateLayout L) {
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t k = i; k < L.first_cells; k += stride) {
    uint64_t key = state[L.first_keys_off + k];
    if (state[L.snap_off + k] != key || key == 0x7fffffffffffffffull) state[L.selval_off + k] = 0;
  }
  for (uint64_t k = i; k < L.last_cells; k += stride) {
    uint64_t key = state[L.last_keys_off + k];
    if (state[L.snap_off + L.first_cells + k] != key || key == 0x8000000000000000ull) state[L.selval_off + L.first_cells + k] = 0;
  }
}

// Multi-GPU: every rank all-gathers the exchange region state[0, exch_words) of all ranks (ONE collective)
// and merges the copies locally, section by section: counts / integer sums wrap-add, f64 sums add in rank
// order (deterministic), min / max keys, and for FIRST / LAST the value of the rank holding the best key.
__global__ void k_merge_gathered(uint64_t *state, StateLayout L, const uint64_t *gathered, uint32_t n_ranks,
                                 uint64_t exch_words) {
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  const uint64_t min_plain = L.first_keys_off - L.min_off, max_plain = L.last_keys_off - L.max_off;
  for (uint64_t k = i; k < L.sum_i64_len; k += stride) {
    uint64_t acc = 0;
    for (uint32_t r = 0; r < n_ranks; r++) acc += gathered[r * exch_words + L.sum_i64_off + k];
    state[L.sum_i64_off + k] = acc;
  }
  for (uint64_t k = i; k < L.sum_f64_len; k += stride) {
    double acc = 0.0;
    for (uint32_t r = 0; r < n_ranks; r++) acc += __longlong_as_double((long long)gathered[r * exch_words + L.sum_f64_off + k]);
    state[L.sum_f64_off + k] = (uint64_t)__double_as_longlong(acc);
  }
  for (uint64_t k = i; k < min_plain; k += stride) {
    int64_t acc = INT64_MAX;
    for (uint32_t r = 0; r < n_ranks; r++) { int64_t v = (int64_t)gathered[r * exch_words + L.min_off + k]; acc = v < acc ? v : acc; }
    state[L.min_off + k] = (uint64_t)acc;
  }
  for (uint64_t k = i; k < max_plain; k += stride) {
    int64_t acc = INT64_MIN;
    for (uint32_t r = 0; r < n_ranks; r++) { int64_t v = (int64_t)gathered[r * exch_words + L.max_off + k]; acc = v > acc ? v : acc; }
    state[L.max_off + k] = (uint64_t)acc;
  }
  for (uint64_t k = i; k < L.first_cells; k += stride) {
    int64_t bk = INT64_MAX; uint64_t bv = 0;
    for (uint32_t r = 0; r < n_ranks; r++) {
      int64_t key = (int64_t)gathered[r * exch_words + L.first_keys_off + k];
      if (key < bk) { bk = key; bv = gathered[r * exch_words + L.selval_off + k]; }
    }
    state[L.first_keys_off + k] = (uint64_t)bk;
    state[L.selval_off + k] = bv;
  }
  for (uint64_t k = i; k < L.last_cells; k += stride) {
    int64_t bk = INT64_MIN; uint64_t bv = 0;
    for (uint32_t r = 0; r < n_ranks; r++) {
      int64_t key = (int64_t)gathered[r * exch_words + L.last_keys_off + k];
      if (key > bk) { bk = key; bv = gathered[r * exch_words + L.selval_off + L.first_cells + k]; }
    }
    state[L.last_keys_off + k] = (uint64_t)bk;
    state[L.selval_off + L.first_cells + k] = bv;
  }
}

// Per output column: which state arrays feed it.
struct OutCol {
  uint64_t count_off;  // counts of the source column
  uint64_t src_off;    // sum / min key / max key / exported first-or-last key
  uint64_t val_off;    // FIRST/LAST: exported values
  uint8_t agg;         // single TSKV_AGG_* bit
  uint8_t phys_type;
  uint8_t pad[6];
};

// Dense result: 8-byte value + Arrow LSB-first validity per cell (one warp packs 32 bits).
__global__ void k_finalize(const uint64_t *state, const OutCol *outs, uint32_t n_out, uint64_t n_cells,
                           uint64_t bitmap_stride, uint64_t *values, uint8_t *validity) {
  const OutCol oc = outs[blockIdx.y];
  uint64_t cell = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  bool valid = false;
  uint64_t v = 0;
  if (cell < n_cells) {
    uint64_t cnt = state[oc.count_off + cell];
    switch (oc.agg) {
      case TSKV_AGG_COUNT: v = cnt; valid = true; break;
      case TSKV_AGG_SUM: valid = cnt > 0; if (valid) v = state[oc.src_off + cell]; break;
      case TSKV_AGG_MIN:
      case TSKV_AGG_MAX: valid = cnt > 0; if (valid) v = okey_inv((int64_t)state[oc.src_off + cell], oc.phys_type); break;
      case TSKV_AGG_MEAN:
        valid = cnt > 0;
        if (valid) {  // src = f64 sum (f64 columns) or exported exact integer sum
          double d = __longlong_as_double((long long)state[oc.src_off + cell]);
          v = (uint64_t)__double_as_longlong(d / (double)cnt);
        }
        break;
      case TSKV_AGG_FIRST: valid = state[oc.src_off + cell] != 0x7fffffffffffffffull; if (valid) v = state[oc.val_off + cell]; break;
      case TSKV_AGG_LAST: valid = state[oc.src_off + cell] != 0x8000000000000000ull; if (valid) v = state[oc.val_off + cell]; break;
      default: break;
    }
    values[(uint64_t)blockIdx.y * n_cells + cell] = v;
  }
  uint32_t bits = __ballot_sync(FULL, valid);
  if ((threadIdx.x & 31) == 0 && (cell >> 3) < bitmap_stride)
    *reinterpret_cast<uint32_t *>(validity + (uint64_t)blockIdx.y * bitmap_stride + (cell >> 3)) = bits;
}

// ------------------------------------------------------------------------------------------------
// upload-time statistics: min / max timestamp of the arena (the reference keeps them per page in
// PageMeta.statistics, written at flush time: tsm/page.rs:212-231). One lane per time page.
__global__ void k_time_bounds(const uint8_t *arena, const tskv_page_desc *descs, const uint32_t *cg_time_page,
                              uint32_t n_cg, long long *bounds /* [0]=min [1]=max */,
                              tskv_time_range *cg_bounds /* per column group (min > max: no timestamps), may be null */) {
  uint32_t cg = blockIdx.x * blockDim.x + threadIdx.x;
  long long lo = INT64_MAX, hi = INT64_MIN;
  if (cg < n_cg) {
    const tskv_page_desc d = descs[cg_time_page[cg]];
    if (kind_status(d.reserved) == TSKV_OK && d.reserved != DK_ALLNULL) {
      PageView pv;
      pv.open(arena, d);
      BitCursor bits;
      bits.init(pv.bitset);
      DeltaCursor<-1> cur;
      if (cur.open(pv, d.reserved) == TSKV_OK) {
        for (uint32_t r = 0; r < d.num_values; r++) {
          if (!bits.next(r)) { if (r == 0) cur.skip_first_if_s8b_sc(); continue; }
          long long t = (long long)cur.next();
          if (cur.exhausted) break;
          lo = t < lo ? t : lo;
          hi = t > hi ? t : hi;
        }
      }
    }
  }
  if (cg_bounds && cg < n_cg) cg_bounds[cg] = tskv_time_range{lo, hi};
  for (int o = 16; o; o >>= 1) {
    long long l2 = (long long)shfl_xor_u64((uint64_t)lo, o), h2 = (long long)shfl_xor_u64((uint64_t)hi, o);
    lo = l2 < lo ? l2 : lo;
    hi = h2 > hi ? h2 : hi;
  }
  if ((threadIdx.x & 31) == 0 && lo <= hi) {
    atomicMin(bounds, lo);
    atomicMax(bounds + 1, hi);
  }
}

}  // namespace tskv
