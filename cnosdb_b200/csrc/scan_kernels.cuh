// scan_kernels.cuh — sm_90a kernels of the tskv scan path:
//   k_worklist : series selection -> work list in fixed (kind bin, column, narrow flag) bucket regions
//       (replaces get_series_id_by_filter's consumer side, tskv/src/reader/iterator.rs:915-929 +
//       SeriesGroupBatchReaderFactory::create :123-264); k_select_ids / k_select_cg: slot of every column group
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
  // bucket regions of the work list (k_worklist): bucket (bin, column, narrow flag) holds region_fill[k] items from
  // region_start[k] on, k = (bin * n_cols + column) * WL_SUB + narrow flag
  const uint32_t *region_start;
  const uint32_t *region_fill;
  const ColState *cols;
  uint64_t *state;
  uint32_t *task_counter;       // [N_BINS] dynamic chunk schedulers
  int32_t *status;              // first error (0 = ok)
  unsigned long long *err_page; // page of the first error
  unsigned long long *stats;    // [0] points decoded, [1] rows in range
  tskv_time_range ranges[MAX_RANGES];
  uint32_t n_ranges;
  // Labelled edge scans (tskvgpu_scan_prepare_labels; 0 for every other scan): the output buckets per group. Edge bucket
  // b then aggregates into output bucket labels[b] < cell_buckets of its group (bucket_cell); the labels follow the
  // n_buckets + 1 edges in the edge table's buffer. (A field in the padding after n_ranges, read only by the EDGES kernels
  // and the merge pass: the tumbling kernels' parameters keep their offsets and their code stays as it was.)
  uint32_t cell_buckets;
  int64_t width;         // <= 0: single bucket
  int64_t origin_mod;    // origin % width; a sliding scan's panes: origin % window, which may lie outside (-width, width)
  // Rows whose dividend t - origin_mod + width does not wrap: [wrap_lo, floor_cap] (set by the host; a tumbling scan has
  // wrap_lo = INT64_MIN). Floor-regime buckets end at floor_cap; rows below wrap_lo are located one by one.
  int64_t floor_cap, wrap_lo;
  int64_t first_bucket_start;
  // Explicit time-bucket edges (tskvgpu_scan_prepare_edges; null for every other scan): bucket b is [edges[b], edges[b + 1]),
  // n_buckets + 1 strictly increasing timestamps. width, origin_mod, floor_cap and wrap_lo are then unused (width = 0).
  const int64_t *edges;
  uint32_t n_buckets;  // time buckets of the grid (edge scans: edge buckets; cell_buckets: a labelled scan's output buckets)
  uint32_t group_by_series;
  uint64_t n_cells;
  // GROUP BY tags: group of every slot, < n_groups with n_groups * cell_buckets < 2^32 (host-checked); null otherwise
  const uint32_t *slot_group;
  // first/last tie-break key. slot_bits == 0 (one slot per cell): key = timestamp itself.
  // Otherwise key = rel << slot_bits | slot with rel = t - key_base(bucket): t - (bucket_start - width) in (0, 2*width)
  // for tumbling scans, t - edges[b] + 1 in [1, edges[b + 1] - edges[b]] for edge scans and t - rel_base for unbucketed
  // ones; the host checked the bit budget.
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
// itself, GROUP BY bucket the one group. Read once per page. A group holds n_buckets cells, or cell_buckets in a labelled
// edge scan (EDGES: the kernels of an edge scan, the only ones that read cell_buckets).
template <bool EDGES>
__device__ __forceinline__ uint64_t group_cell_base(const ScanParams &P, uint32_t slot) {
  if constexpr (EDGES) {
    const uint64_t per = P.cell_buckets ? P.cell_buckets : P.n_buckets;
    if (P.slot_group) return __ldg(P.slot_group + slot) * per;
    return P.group_by_series ? slot * per : 0;
  }
  if (P.slot_group) return (uint64_t)__ldg(P.slot_group + slot) * P.n_buckets;
  return P.group_by_series ? (uint64_t)slot * P.n_buckets : 0;
}

// Output bucket of bucket b within its group: labels[b] for a labelled edge scan, b for every other scan. Every bucket ->
// cell step goes through here. `need`: the lane uses the result (a lane that does not skips the load).
template <bool EDGES>
__device__ __forceinline__ uint32_t bucket_cell(const ScanParams &P, uint32_t b, bool need = true) {
  if constexpr (EDGES) {
    const uint32_t *labels = reinterpret_cast<const uint32_t *>(P.edges + P.n_buckets + 1);
    return (P.cell_buckets && need) ? __ldg(labels + b) : b;
  }
  return b;
}

// ------------------------------------------------------------------------------------------------
// selection / compaction
// ------------------------------------------------------------------------------------------------
// Series id -> rank among the page set's distinct ids (FULL: the page set does not hold the id). A page set whose ids
// are dense (plan_series_map) has a direct table rank_of[id - min_id]: one load instead of a binary search of ~20
// dependent steps over the sorted ids.
struct SeriesIndex {
  const uint32_t *sorted;   // the page set's distinct series ids, ascending
  const uint32_t *rank_of;  // [span] rank of id min_id + k, FULL for an id without series (null: binary search)
  uint32_t n, min_id, span;
};
__device__ __forceinline__ uint32_t series_rank(const SeriesIndex &S, uint32_t id) {
  if (S.rank_of) {
    const uint32_t k = id - S.min_id;  // ids below min_id wrap past the span
    return k < S.span ? __ldg(S.rank_of + k) : FULL;
  }
  uint32_t lo = 0, hi = S.n;
  while (lo < hi) {
    const uint32_t mid = (lo + hi) >> 1;
    if (__ldg(S.sorted + mid) < id) lo = mid + 1; else hi = mid;
  }
  return lo < S.n && __ldg(S.sorted + lo) == id ? lo : FULL;
}

// Series selection -> slot of every column group, in two steps: one thread per SELECTED id finds the id's rank among
// the page set's series and writes its position in the selection list to rank_slot[rank] (memset to -1 before); then
// one thread per column group gathers rank_slot[rank of its series].
// (Round 1 searched the selection list once per column group: 10 x the dependent loads for a 10 % selection.)
__global__ void k_select_ids(const SeriesIndex S, const uint32_t *series_ids, uint32_t n_series, int32_t *rank_slot) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_series) return;
  const uint32_t rank = series_rank(S, __ldg(series_ids + i));
  if (rank != FULL) rank_slot[rank] = (int32_t)i;
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

// The reader counters of a scan pass, in unsigned long long words: pages read, their bytes, the bytes each bin's fused
// kernel reads, and the field pages that statistics pruning dropped.
constexpr uint32_t CTR_PAGES = 0, CTR_BYTES = 1, CTR_BIN_BYTES = 2, CTR_PRUNED = CTR_BIN_BYTES + N_BINS,
                   N_COUNTERS = CTR_PRUNED + 1;

// Statistics pruning (filter_column_groups, tskv/src/reader/chunk.rs:12-50 with the column group's time_range(),
// tsm/column_group.rs:9-17): a group whose [min_ts, max_ts] overlaps none of the query's time ranges is dropped by the
// work-list walk, so its pages are neither gathered nor decoded.
struct PruneRanges {
  tskv_time_range r[MAX_RANGES];
  uint32_t n;
  uint32_t pad;
};

// ------------------------------------------------------------------------------------------------
// Work list driven by the SELECTION: 2^split_log2 threads per selected series walk that series' column groups (thread j
// of a series takes groups j, j + S, j + 2S, ... of it) and their field pages, so the cost follows the selection (C4:
// 10 % of the series) instead of the page set, and a series with thousands of groups is not walked by one thread.
// Items go to buckets (decode-kind bin, query column, narrow flag): the fused kernels need warps that are homogeneous in
// codec and, for GROUP BY bucket, in column, and a (bin, column) bucket is split in two by the page's narrow flag
// (WL_SUB buckets, ScanParams.page_narrow) so that a chunk is uniformly narrow or wide. Every bucket owns a fixed region
// of the work list, laid out by the host at prepare (plan_worklist_regions): it starts on a multiple of 32 and holds the
// page set's field pages of the bucket's bin, column id and narrow flag, an upper bound for any selection. So one
// kernel places every item without a pass over all blocks' counts in between, and no chunk of 32 items straddles two
// buckets. Inside a bucket the order is arbitrary. Outputs:
// work_page / work_slot / work_qcol (bit 7 = "brings the column group's time page": the first selected field page of
// each value class of a group), the buckets' fill counts, the reader counters (the reference's reader metrics,
// column_group/mod.rs:141-193, split per decode-kind bin), statistics pruning.
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
  SeriesIndex series;            // the page set's series ids -> ranks
  const uint32_t *series_ids;    // the selection (null: every series, slot = rank)
  uint32_t n_sel;                // walk indices: selected ids, or n_set_series
  uint32_t split_log2;           // log2 of the threads per walk index (plan_walk_split)
  // GROUP BY tags: walk index i walks slot walk[i], the slots stably sorted by group, so that the items of a (bin,
  // column) bucket come group by group and a warp's 32 pages mostly share a group (null: walk index i walks slot i)
  const uint32_t *walk;
  const ColState *cols;
  uint32_t n_cols;
  const tskv_time_range *cg_bounds;  // statistics pruning (null: none)
  PruneRanges prune;
  const uint8_t *cg_merge;       // column groups of overlapping chunks go through the merge pass
  const int64_t *page_stats;     // value-statistics pruning against `preds` (null: none)
  PredicateSet preds;
  const uint32_t *region_start;  // [N_BINS * n_cols * WL_SUB + 1] first work-list index of every bucket's region
  uint32_t *bucket_fill;         // [N_BINS * n_cols * WL_SUB] items placed in each bucket (zeroed by k_init_state)
  uint32_t *work_page, *work_slot;
  uint8_t *work_qcol;
  unsigned long long *counters;  // [N_COUNTERS] CTR_*
  int32_t *status;
};

// Work-list bucket of a page: (bin, query column, narrow flag).
__device__ __forceinline__ uint32_t worklist_key(const WorkListArgs &A, uint32_t page, uint32_t bin, uint32_t qc) {
  return (bin * A.n_cols + qc) * WL_SUB + ((A.page_narrow && A.page_narrow[page]) ? 1u : 0u);
}

// Walks the items of column groups j, j + S, ... of selected series i (S = 2^split_log2); everything per column group
// stays inside one thread. F(page, bin, qcol, with_time, desc, first_in_group, time page).
template <typename F>
__device__ __forceinline__ void worklist_walk(const WorkListArgs &A, uint32_t i, uint32_t j, bool count_stats, F &&emit) {
  uint32_t rank = i;
  if (A.series_ids) {
    rank = series_rank(A.series, __ldg(A.series_ids + i));
    if (rank == FULL) return;  // a selected id this page set does not hold
  }
  const uint32_t c0 = __ldg(A.rank_cg_start + rank), c1 = __ldg(A.rank_cg_start + rank + 1);
  for (uint32_t k = c0 + j; k < c1; k += 1u << A.split_log2) {
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
    // The time page of a column group is brought along (PCIe gather, CRC check) by the first selected field page of the
    // group IN EACH DECODE-KIND BIN: the bins' gathers and fused kernels run on different streams, so a bin must not rely
    // on another bin having copied it (an i64 and an f64 field of one series land in two bins). Field pages of a group
    // share its time class, so "same bin" is "same value class".
    uint32_t seen_classes = 0;  // value classes that already brought the time page
    bool any = false;
    for (uint64_t p = (uint64_t)tp + 1; p < end; p++) {
      const tskv_page_desc d = A.descs[p];
      const int qc = find_qcol(A.cols, A.n_cols, d.column_id);
      if (qc < 0) continue;
      if (!in_time) {
        if (count_stats) atomicAdd(&A.counters[CTR_PRUNED], 1ull);
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

// The walk, twice over the block's series: first the block's items per bucket and the reader counters (per block in
// shared memory), then - after one atomic per (block, bucket) on the bucket's fill count has reserved the block's share
// of the region - the items' places. Inside a block the items keep the order of the shared-memory cursors, so scans of a
// few blocks place their items in a stable order (float sums of two runs of one scan agree bit for bit); a warp-wide
// reservation per item instead would interleave the warps of a block.
__global__ void __launch_bounds__(WL_THREADS) k_worklist(const WorkListArgs A) {
  extern __shared__ uint32_t s_hist[];  // [2][N_BINS * n_cols * WL_SUB]: block counts -> block bases, and the running cursors
  __shared__ unsigned long long s_pages, s_bytes[N_BINS];
  const uint32_t n_buckets = N_BINS * A.n_cols * WL_SUB;
  uint32_t *s_base = s_hist, *s_cur = s_hist + n_buckets;
  for (uint32_t k = threadIdx.x; k < 2 * n_buckets; k += WL_THREADS) s_hist[k] = 0;
  if (threadIdx.x == 0) s_pages = 0;
  if (threadIdx.x < N_BINS) s_bytes[threadIdx.x] = 0;
  __syncthreads();
  const uint32_t t = blockIdx.x * WL_THREADS + threadIdx.x, i = t >> A.split_log2, j = t & ((1u << A.split_log2) - 1);
  const uint32_t slot = (i < A.n_sel && A.walk) ? __ldg(A.walk + i) : i;
  if (i < A.n_sel)
    worklist_walk(A, slot, j, true, [&](uint32_t page, uint32_t bin, uint32_t qc, bool, const tskv_page_desc &d, bool first_in_group, uint32_t tp) {
      atomicAdd(&s_base[worklist_key(A, page, bin, qc)], 1u);
      // the reader metrics (page_read_count / page_read_bytes) count the time page once per column group
      unsigned long long bytes = d.size, pages = 1;
      if (first_in_group) { bytes += A.descs[tp].size; pages += 1; }
      atomicAdd(&s_bytes[bin], bytes);
      atomicAdd(&s_pages, pages);
    });
  __syncthreads();
  for (uint32_t k = threadIdx.x; k < n_buckets; k += WL_THREADS)
    if (s_base[k]) s_base[k] = A.region_start[k] + atomicAdd(&A.bucket_fill[k], s_base[k]);
  if (threadIdx.x == 0 && s_pages) atomicAdd(&A.counters[CTR_PAGES], s_pages);
  if (threadIdx.x < N_BINS && s_bytes[threadIdx.x]) {
    atomicAdd(&A.counters[CTR_BYTES], s_bytes[threadIdx.x]);
    atomicAdd(&A.counters[CTR_BIN_BYTES + threadIdx.x], s_bytes[threadIdx.x]);
  }
  __syncthreads();
  if (i < A.n_sel)
    worklist_walk(A, slot, j, false, [&](uint32_t page, uint32_t bin, uint32_t qc, bool with_time, const tskv_page_desc &, bool, uint32_t) {
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
                               const uint8_t *work_qcol, const uint32_t *region_start, const uint32_t *bucket_fill,
                               uint32_t per_bin, int bin) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t warps = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t k = bin * per_bin; k < (bin + 1) * per_bin; k++)  // the bin's bucket regions
  for (uint32_t w = region_start[k] + ((blockIdx.x * blockDim.x + threadIdx.x) >> 5), n = region_start[k] + bucket_fill[k]; w < n; w += warps) {
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
             const uint32_t *work_page, const uint8_t *work_qcol, const uint32_t *region_start, const uint32_t *bucket_fill,
             uint32_t per_bin, int bin,
             const uint32_t *crc_tables /* [8][256] */, int32_t *status, unsigned long long *err_page) {
  __shared__ uint32_t s_t[8][256];
  for (uint32_t i = threadIdx.x; i < 2048; i += blockDim.x) s_t[i >> 8][i & 255] = crc_tables[i];
  __syncthreads();
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t k = bin * per_bin; k < (bin + 1) * per_bin; k++)  // the bin's bucket regions
  for (uint32_t w = region_start[k] + blockIdx.x * blockDim.x + threadIdx.x, n = region_start[k] + bucket_fill[k]; w < n; w += stride) {
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

// Base of the FIRST / LAST tie-break key of bucket `bucket` (ScanParams::slot_bits): rel = t - base > 0. EDGES: an edge
// scan (P.edges != null; a template argument so that the tumbling kernels hold none of its code).
template <bool EDGES>
__device__ __forceinline__ uint64_t key_base(const ScanParams &P, int64_t bucket) {
  if constexpr (EDGES) return (uint64_t)__ldg(P.edges + bucket) - 1;
  return P.width > 0 ? (uint64_t)P.first_bucket_start + (uint64_t)(bucket - 1) * (uint64_t)P.width : (uint64_t)P.rel_base;
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

// Warp-converged flush of run partials into the global state. `active` lanes carry a finished
// run for cell `gcell` (= qcol * n_cells + cell). When every flushing lane targets the same cell
// (the common lock-step case of GROUP BY bucket) the partials are combined with a butterfly first
// and one lane issues the atomics.
template <bool SEL, bool EDGES>
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
    const uint64_t base = key_base<EDGES>(P, bucket);
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
// EDGES (an edge scan, P.edges): bucket b is [edges[b], edges[b + 1]) - floor semantics at every time, no wrapped regime.
template <bool EDGES>
__device__ __forceinline__ bool locate_bucket(const ScanParams &P, int64_t t, BucketState &b) {
  if constexpr (EDGES) {
    const int64_t *E = P.edges;
    if (b.valid && t > b.hi && b.idx + 1 < P.n_buckets) {  // the next bucket: [b.hi + 1, edges[b.idx + 2])
      const int64_t e2 = __ldg(E + b.idx + 2);
      if (t < e2) {
        b.lo = b.hi + 1;
        b.hi = e2 - 1;
        b.idx += 1;
        return true;
      }
    }
    if (t < __ldg(E) || t >= __ldg(E + P.n_buckets)) return false;
    uint32_t lo = 0, hi = P.n_buckets - 1;  // the last bucket whose start is <= t
    while (lo < hi) {
      const uint32_t mid = (lo + hi + 1) >> 1;
      if (__ldg(E + mid) <= t) lo = mid; else hi = mid - 1;
    }
    b.lo = __ldg(E + lo);
    b.hi = __ldg(E + lo + 1) - 1;
    b.idx = lo;
    b.valid = true;
    b.floor_regime = true;
    return true;
  }
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

// Upper bound of bucket idx + 1, for a floor-regime bucket idx that ends at hi: locate_bucket's next-bucket step (the
// next edge, or hi + width cut at floor_cap). hi itself when no bucket follows in that regime.
template <bool EDGES>
__device__ __forceinline__ int64_t next_bucket_hi(const ScanParams &P, uint32_t idx, int64_t hi) {
  if (idx + 1 >= P.n_buckets) return hi;
  if constexpr (EDGES) return __ldg(P.edges + idx + 2) - 1;
  const uint64_t room = (uint64_t)P.floor_cap - (uint64_t)hi;
  return (int64_t)((uint64_t)hi + (room < (uint64_t)P.width ? room : (uint64_t)P.width));
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

// The row engine of the fused scan: one chunk of <= 32 work items, one lane per field page, the whole warp converged.
// Per lane:
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

// Pass 2 of TSKV_AGG_M2 (k_scan_m2): a run's ValueAcc holds sum(d) in `sum` and sum(d^2) in `sum_hi` (f64 bits) with
// d = (double)x - shift, shift = the run's cell mean from pass 1 (k_m2_prep), held as f64 bits in `kmin` (unused by the
// pass). Integers convert to f64 as DataFusion's variance does.
template <int VK>
__device__ __forceinline__ void m2_add(ValueAcc<VK> &va, uint64_t v, uint8_t pt) {
  const double shift = __longlong_as_double((long long)va.kmin);
  double x;
  if (VK == VK_GOR || pt == TSKV_PT_F64) x = __longlong_as_double((long long)v);
  else if (pt == TSKV_PT_I64) x = (double)(int64_t)v;
  else x = (double)v;
  const double d = x - shift;
  va.sum = (uint64_t)__double_as_longlong(__longlong_as_double((long long)va.sum) + d);
  va.sum_hi = __double_as_longlong(__longlong_as_double((long long)va.sum_hi) + d * d);
}

// sum(d) / sum(d^2) of one run (pass 2) into the partial table: the CTA's shared-memory table (s_sum / s_hi) or the
// global state (sum_off / sumhi_off of the pass-2 column table, see M2Col).
__device__ __forceinline__ void table_update_m2(const ScanParams &P, uint64_t *stab, const ColState &cs, uint64_t cell,
                                                uint64_t sd, uint64_t sd2) {
  const bool sm = P.use_smem != 0;
  uint64_t *tab = sm ? stab : P.state;
  atomicAdd(reinterpret_cast<double *>(tab + (sm ? cs.s_sum : cs.sum_off) + cell), __longlong_as_double((long long)sd));
  atomicAdd(reinterpret_cast<double *>(tab + (sm ? cs.s_hi : cs.sumhi_off) + cell), __longlong_as_double((long long)sd2));
}

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

// M2 (pass 2 of TSKV_AGG_M2): the staged quantities are count | sum(d) | sum(d^2), both sums f64.
template <int VK, int NS, bool M2 = false>
__device__ __forceinline__ void reduce_staged(const ScanParams &P, uint64_t *stab, uint64_t *stage, uint32_t n_slots) {
  __syncwarp();
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t s = lane & (NS - 1), g = lane / NS;
  const uint64_t meta = stage[NS * FLUSH_Q * 32 + s];  // (query column << 32) | cell
  const uint32_t qcol = (uint32_t)(meta >> 32);
  const ColState &cs = P.cols[s < n_slots ? qcol : 0];
  if constexpr (M2) {
    uint64_t cnt = 0;
    double sd = 0.0, sd2 = 0.0;
    const uint64_t *base = stage + (size_t)s * FLUSH_Q * 32;
#pragma unroll
    for (int i = 0; i < NS; i++) {
      const uint32_t src = g * NS + ((i + s) & (NS - 1));
      cnt += base[src];
      sd += __longlong_as_double((long long)base[32 + src]);
      sd2 += __longlong_as_double((long long)base[64 + src]);
    }
#pragma unroll
    for (int o = NS; o < 32; o <<= 1) {
      cnt += shfl_xor_u64(cnt, o);
      sd += __longlong_as_double((long long)shfl_xor_u64((uint64_t)__double_as_longlong(sd), o));
      sd2 += __longlong_as_double((long long)shfl_xor_u64((uint64_t)__double_as_longlong(sd2), o));
    }
    if (lane < n_slots && cnt)
      table_update_m2(P, stab, cs, (uint64_t)(uint32_t)meta, (uint64_t)__double_as_longlong(sd), (uint64_t)__double_as_longlong(sd2));
    __syncwarp();
    return;
  }
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

// This lane's partial (identities unless `live`) into its column of staging slot `seq`.
template <int VK, bool M2 = false>
__device__ __forceinline__ void stage_lane(uint64_t *stage, uint32_t seq, bool live, const ValueAcc<VK> &va) {
  uint64_t *q = stage + (size_t)seq * FLUSH_Q * 32 + (threadIdx.x & 31);
  q[0] = live ? va.count : 0;
  q[32] = live ? va.sum : 0;  // 0 bits == +0.0
  if (VK != VK_GOR || M2) q[64] = live ? (uint64_t)va.sum_hi : 0;
  if constexpr (!M2) {
    q[96] = live ? (uint64_t)va.kmin : (uint64_t)INT64_MAX;
    q[128] = live ? (uint64_t)va.kmax : (uint64_t)INT64_MIN;
  }
}

// Every lane parks its partial (identities unless `live`) in staging slot `seq`, the lane `meta_lane` records the slot's
// (query column << 32) | cell, and every NS slots the warp reduces them. Called by all 32 lanes.
template <int VK, int NS, bool M2 = false>
__device__ __forceinline__ void stage_partial(const ScanParams &P, uint64_t *stab, uint64_t *stage, uint32_t &seq, bool live,
                                              const ValueAcc<VK> &va, bool meta_lane, uint64_t gcell) {
  stage_lane<VK, M2>(stage, seq, live, va);
  if (meta_lane) stage[NS * FLUSH_Q * 32 + seq] = gcell;
  if (++seq == NS) {
    reduce_staged<VK, NS, M2>(P, stab, stage, seq);
    seq = 0;
  }
}

// Flush of one finished run per flushing lane (no FIRST/LAST). `seq` = staged slots in use (warp-uniform). M2: pass 2 of
// TSKV_AGG_M2 (sum(d) / sum(d^2) partials, m2_add).
template <int VK, int NS, bool M2 = false>
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
    stage_partial<VK, NS, M2>(P, stab, stage, seq, active && va.count, va, (int)lane == leader, lcell);
  } else if (active && va.count) {  // lanes on different cells (GROUP BY series, unaligned pages): one update each
    if constexpr (M2) table_update_m2(P, stab, P.cols[qcol], cell, va.sum, (uint64_t)va.sum_hi);
    else table_update(P, stab, P.cols[qcol], cell, mask, VK == VK_GOR || (VK == VK_GEN && pt == TSKV_PT_F64), va.count, va.sum,
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

// Edge scans, RLE row space: rows of the page from the row at time t (>= edges[b]) on that lie in bucket b, i.e. before
// edges[b + 1] (0: the bucket ends before t). A bucket past the last one returns 1, so that the caller's step stops there
// and reports TSKV_ERR_BUCKET_RANGE.
__device__ __forceinline__ uint32_t edge_rows(const ScanParams &P, uint32_t b, uint64_t t, uint64_t delta, double inv) {
  if (b >= P.n_buckets) return 1u;
  const int64_t end = __ldg(P.edges + b + 1);
  return (int64_t)t < end ? rle_rows_within((uint64_t)end - 1 - t, delta, inv, 0xffffffffu) : 0u;
}

// Time cursor of TK_GEN: any time codec straight from global memory, with the time validity bitmap. (The bitmap state
// lives in the cursor so that the other time classes declare nothing they do not use.)
struct GenTimeCursor : DeltaCursor<-1, BeStream> {
  const uint32_t *bm = nullptr;  // time validity bitmap
  uint32_t word = 0;             // its word of row `row`
  bool none = false;             // the page has no valid time row
};

// TK = the time class: RLE timestamps in closed form, simple8b ones staged through a time ring, or generic (TK_GEN: time
// pages that are raw-encoded, hold NULLs or fail to decode - nothing the reference's writer produces, flush rejects a
// time column with nulls, mem_cache/series_data.rs:303-340) read from global memory. A NULL-time row fails
// is_not_null(time) like a row the row filter drops: its keep bit is cleared, its value is still decoded. It keeps the
// timestamp of the row before it (leading NULLs: of the first valid row), so it never cuts a segment of its own.
// NARROW (simple8b integer values, no FIRST / LAST): every page of the chunk is narrow (ScanParams.page_narrow), so the
// values are decoded and accumulated in 32-bit arithmetic (S8bCursor::next32, ValueAcc::add32).
// M2 (k_scan_m2, pass 2 of TSKV_AGG_M2; never with SEL or NARROW): the same rows, segments and runs, but a run sums
// d = x - (its cell's pass-1 mean) and d^2 (m2_add) instead of count / sum / min / max, and counts no points or rows.
// The uniform schedule is left to the segment loop, which gives the same rows.
template <int TK, int VK, bool SEL, bool NARROW, bool EDGES, bool M2 = false>
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
  // TK_S8B: timestamps staged through the time ring; TK_GEN: GenTimeCursor
  typename std::conditional<TK == TK_GEN, GenTimeCursor, S8bCursor<false>>::type tcur;
  uint64_t rle_t0 = 0, rle_delta = 0;          // TK_RLE: t(row) = rle_t0 + row * rle_delta (wrapping), closed form
  double rle_inv = 0.0;
  typename std::conditional<VK == VK_S8B, S8bCursor<true>, DeltaCursor<-1, SeqStream>>::type vcur_d;
  GorillaRing vcur_g;
  const uint32_t *vbm = nullptr;  // value validity bitmap, 32 rows per word
  const uint32_t *keepw = nullptr;  // row-filter keep bits of the column group (k_row_filter), or null
  bool allnull = false;
  int64_t pend_t = 0;  // timestamp of row `row`

  if constexpr (TK == TK_S8B) tcur.reset(tslot);
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
    tskv_status st = kind_status(vd.reserved);  // (RLE / simple8b time pages always decode)
    uint32_t st_page = page;
    if constexpr (TK == TK_GEN) {  // the time page's error comes first
      if (kind_status(td.reserved) != TSKV_OK) { st = kind_status(td.reserved); st_page = tpage; }
    }
    if (part != 0 && (!split || r0 >= page_rows)) {
      // nothing for this lane: the page ends before this part, or part 0's lane decodes all of it
    } else if (st != TSKV_OK) {
      report_error(P, st, st_page);
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
      } else if constexpr (TK == TK_S8B) {
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
      if constexpr (TK == TK_GEN) {
        if (td.reserved == DK_ALLNULL) n_rows = 0;  // no time values: every row fails is_not_null(time)
        tcur.bm = reinterpret_cast<const uint32_t *>(tpv.bitset);
      }
      if (st == TSKV_OK && n_rows) {
        if (TK == TK_RLE) {
          pend_t = (int64_t)(rle_t0 + (uint64_t)r0 * rle_delta);
        } else if constexpr (TK == TK_GEN) {
          uint32_t f = 0, w = 0;  // the first valid time row: its timestamp is row 0's (rows before it are NULL)
          while (f < n_rows && (w = __ldg(tcur.bm + (f >> 5))) == 0) f += 32;
          if (f < n_rows) f += __ffs(w) - 1;
          tcur.none = f >= n_rows;
          if (f == 0) {
            pend_t = (int64_t)tcur.next();
          } else if (!tcur.none) {  // peek: row f takes the value when the row loop reaches it
            tcur.skip_first_if_s8b_sc();
            DeltaCursor<-1, BeStream> peek = tcur;
            pend_t = (int64_t)peek.next();
          }
          tcur.word = __ldg(tcur.bm);
        } else if (part == 0) {
          pend_t = (int64_t)tcur.next();  // the first value: no ring access (cursors.cuh)
        } else {
          pend_t = (int64_t)tcur.v;
        }
      }
      if (st != TSKV_OK) { report_error(P, st, st == TSKV_ERR_BITSET_MISMATCH ? tpage : page); n_rows = 0; }
    }
  }
  const bool to_page_end = n_rows == page_rows;  // this lane reaches the end of the page's streams
  ring_drain();  // the rings' initial fills have landed before the first step (once per page)

  static_assert(!NARROW || (VK == VK_S8B && !SEL), "narrow chunks: simple8b integer values, no FIRST / LAST");
  static_assert(!M2 || (!SEL && !NARROW), "M2 pass: no FIRST / LAST, wide arithmetic");
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
  const uint64_t group_base = SEL ? 0 : group_cell_base<EDGES>(P, slot);
  uint32_t staged = 0;  // staged flush slots in use (warp-uniform)

  // Finished runs of the flushing lanes -> partial tables.
  auto flush_now = [&](bool flush) {
    if constexpr (M2) {
      flush_runs<VK, NS, true>(P, stab, stage, staged, flush, qcol, group_base + bucket_cell<EDGES>(P, run_idx, flush), pt, mask, va);
      return;
    }
    if (flush) va.fold(pt, NARROW);
    if (SEL) {
      if (__any_sync(FULL, flush)) {
        acc.count = va.count; acc.sum = va.sum; acc.sum_hi = va.sum_hi; acc.kmin = va.kmin; acc.kmax = va.kmax;
        const uint32_t fslot = have_item ? __ldg(P.work_slot + item) : 0u;
        warp_flush<SEL, EDGES>(P, stab, flush, qcol, group_cell_base<EDGES>(P, fslot) + bucket_cell<EDGES>(P, run_idx, flush),
                               (int64_t)run_idx, pt, mask, acc, fslot);
      }
    } else {
      flush_runs<VK, NS>(P, stab, stage, staged, flush, qcol, group_base + bucket_cell<EDGES>(P, run_idx, flush), pt, mask, va);
    }
  };
  // One row's value: validity bit, decode (every valid row is decoded - rows outside the time ranges too, the streams
  // are sequential), accumulate when the segment is selected. Returns the value; `vv` = the row holds one.
  auto row_value = [&](bool accumulate, bool &vv, bool &kept) -> uint64_t {
    if ((row & 31) == 0) {  // entering a new bitmap word: take the prefetched one, prefetch the next
      vword = vahead;
      vahead = __ldg(vbm + (row >> 5) + 1);  // reads at most 8 bytes past the bitmap (inside the page)
      if constexpr (TK == TK_GEN) kword = (keepw ? __ldg(keepw + (row >> 5)) : 0xffffffffu) & tcur.word;
      else if (keepw) kword = __ldg(keepw + (row >> 5));
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
        if constexpr (M2) {
          if (accumulate && kept) { va.count++; m2_add(va, v, pt); }
        } else {
          if (accumulate && kept) { va.count++; va.add(v, pt, flip); }
        }
      }
    }
    return v;  // (0 for narrow chunks: only FIRST / LAST use it)
  };
  // The next value, accumulated when `take` (every value is decoded: the streams are sequential).
  auto next_add = [&](bool take) {
    if constexpr (NARROW) {
      const uint32_t v32 = vcur_d.next32();
      if (take) va.add32(v32);
    } else if constexpr (M2) {
      const uint64_t v = VK == VK_GOR ? vcur_g.next() : vcur_d.next();
      if (take) m2_add(va, v, pt);
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
        if ((P.width > 0 || EDGES) && ra < rb1) {
          const int64_t tr = (int64_t)(rle_t0 + (uint64_t)ra * rle_delta);
          if (P.width > 0 && (int64_t)((uint64_t)tr - (uint64_t)P.origin_mod + (uint64_t)P.width) < 0) {
            elig = false;  // truncating-% regime (time_window.rs:184-198): general logic
          } else if (!locate_bucket<EDGES>(P, tr, bk)) {
            report_error(P, TSKV_ERR_BUCKET_RANGE, page);
            n_rows = 0;
          } else {
            bidx = bk.idx;
            nb = rle_rows_within((uint64_t)bk.hi - (uint64_t)tr, rle_delta, rle_inv, 0xffffffffu);
            if (P.width > 0) {  // (edge scans step with edge_rows)
              e_off = (uint64_t)tr + (uint64_t)nb * rle_delta - ((uint64_t)bk.hi + 1);
              q32 = rle_rows_within((uint64_t)P.width, rle_delta, rle_inv, 0xffffffffu) - 1;
              w_rem = (uint64_t)P.width - (uint64_t)q32 * rle_delta;
            }
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
  if (TK == TK_RLE && VK != VK_GEN && !SEL && fast && (P.width > 0 || EDGES) && !P.group_by_series && !M2) {
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
      if (EDGES) {  // edge_rows steps from the row's time
        rle_t0 = shfl_u64(rle_t0, src);
        rle_inv = __longlong_as_double((long long)shfl_u64((uint64_t)__double_as_longlong(rle_inv), src));
      }
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
              if (EDGES) {
                do {
                  bidx++;
                  nb = edge_rows(P, bidx, rle_t0 + (uint64_t)r * rle_delta, rle_delta, rle_inv);
                } while (nb == 0);
              } else {
                do {
                  bidx++;
                  nb = q32 + (e_off < w_rem ? 1u : 0u);
                  e_off = e_off + (uint64_t)nb * rle_delta - (uint64_t)P.width;
                } while (nb == 0);
              }
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
            stage_partial<VK, NS>(P, stab, stage, staged, n_rows && va.count, va, lane == 0, col + bucket_cell<EDGES>(P, bidx));
            va.reset(NARROW);
          }
        }
        row = r;
      }
      row = n_rows;  // nothing is left for the segment loop below
    }
  }

  // ---- Lockstep schedule (simple8b timestamps, GROUP BY bucket / tags / edges / labels, no FIRST / LAST, at most one time
  // range, no tombstones). When all 32 lanes hold rows, start and end at the same row, have the same query column and
  // group, and their first rows lie in one bucket or the next (pages cut into equal parts: C4's jittered pages), the warp
  // walks the rows one at a time in all lanes together and keeps ONE bucket schedule: bucket bidx = [blo, bhi] and the
  // bound bhi2 of the next one. Every lane still decodes and compares its own timestamps. A lane whose row first passes
  // bhi parks its partial of bidx in its column of staging slot `staged` and goes on accumulating bidx + 1 in the same
  // registers; once every lane has crossed, the slot is committed and the schedule steps. This takes the segment head,
  // the alignment reduction and the flush vote off every bucket, and no lane runs a row trip another lane does not need.
  // The lanes' runs and the order of the staged slots are the ones the segment loop makes for such a warp. A row outside
  // [blo, bhi2] (a gap, an empty bucket, the last bucket, time going backwards) or outside the time range, or a decode
  // error at a lane's bucket end, hands the warp to the segment loop at that row, before it is consumed. On C4 the step
  // follows the instructions per row, not the cycles the segment head kept a warp waiting (DESIGN.md §5), so the row is
  // kept lean: one reduction decides the warp's step, every row the walk takes is inside the range (the range's bounds
  // clip the lane's window instead of being tested per row), and a chunk with lanes that hold no rows keeps the segment
  // loop rather than predicating every row on them.
  if constexpr (TK == TK_S8B && VK != VK_GEN && !SEL && !M2) {
    const int64_t tr_lo = P.n_ranges ? P.ranges[0].min_ts : INT64_MIN, tr_hi = P.n_ranges ? P.ranges[0].max_ts : INT64_MAX;
    if ((P.width > 0 || EDGES) && !P.group_by_series && P.n_ranges <= 1 && tr_lo <= tr_hi && !P.has_tomb &&
        __all_sync(FULL, row < n_rows)) {
      const bool located = locate_bucket<EDGES>(P, pend_t, bk) && bk.floor_regime;
      // the first bucket: the earliest of the lanes' (a part that starts on a bucket edge has lanes in the next one too)
      const uint32_t b0 = __reduce_min_sync(FULL, located ? bk.idx : 0xffffffffu);
      const bool agree = located & (pend_t >= tr_lo) & (pend_t <= tr_hi) &
                         (__shfl_sync(FULL, row, 0) == row) & (__shfl_sync(FULL, n_rows, 0) == n_rows) &
                         (__shfl_sync(FULL, qcol, 0) == qcol) &
                         (__shfl_sync(FULL, (uint32_t)group_base, 0) == (uint32_t)group_base) & (bk.idx - b0 <= 1u);
      if (__all_sync(FULL, agree)) {
        const int src = __ffs(__ballot_sync(FULL, bk.idx == b0)) - 1;
        uint32_t bidx = b0;
        int64_t blo = (int64_t)shfl_u64((uint64_t)bk.lo, src), bhi = (int64_t)shfl_u64((uint64_t)bk.hi, src);
        int64_t bhi2 = next_bucket_hi<EDGES>(P, bidx, bhi);
        const uint64_t col = ((uint64_t)qcol << 32) | (uint32_t)group_base;
        int64_t t = pend_t;
        bool crossed = bk.idx != b0;  // this lane's rows have reached bucket bidx + 1
        if (crossed) stage_lane<VK>(stage, staged, false, va);  // (it has no row in bucket bidx)
        // this lane's next row must lie in [wlo, wlo + wspan]: in its bucket or the next one, and inside the range
        int64_t wlo = 0;
        uint64_t wspan = 0;
        auto window = [&]() {
          const int64_t lo = crossed ? bhi + 1 : blo, hi = bhi2 < tr_hi ? bhi2 : tr_hi;
          wlo = lo > tr_lo ? lo : tr_lo;
          wspan = (uint64_t)hi - (uint64_t)wlo;  // (t lies in the window when it is set: never empty)
        };
        window();
        // slot `staged` of bucket bidx is complete: the lanes that have not filled their column there hold identities
        auto commit = [&](bool filled) {
          if (!filled) stage_lane<VK>(stage, staged, false, va);
          if (lane == 0) stage[NS * FLUSH_Q * 32 + staged] = col + bucket_cell<EDGES>(P, bidx);
          if (++staged == NS) {
            reduce_staged<VK, NS>(P, stab, stage, staged);
            staged = 0;
          }
        };
#pragma unroll 1
        while (row < n_rows) {
          const bool up = t > bhi;  // row `row` lies past bucket bidx
          const bool cross = up && !crossed;
          // (the segment loop checks the cursors where a lane's segment ends: here, where the lane crosses)
          const bool bad = (uint64_t)t - (uint64_t)wlo > wspan ||
                           (cross && (cursor_exhausted(tcur) || (VK == VK_GOR ? vcur_g.failed() : cursor_exhausted(vcur_d))));
          // one reduction for the warp's next step: 0 = a lane leaves the schedule, 2 = every lane is past bucket bidx
          const uint32_t step = __reduce_min_sync(FULL, bad ? 0u : up ? 2u : 1u);
          if (step == 0) break;
          if (cross) {
            va.fold(pt, NARROW);
            stage_lane<VK>(stage, staged, va.count != 0, va);
            va.reset(NARROW);
            crossed = true;
            window();
          }
          if (step == 2) {
            commit(true);
            bidx++;
            blo = bhi + 1;
            bhi = bhi2;
            bhi2 = next_bucket_hi<EDGES>(P, bidx, bhi);
            crossed = false;
            window();
          }
          // the next row's timestamp first: its chain runs beside the value's (past the last row this runs one value too
          // far - harmless)
          const int64_t tn = (int64_t)tcur.next();
          bool vv, kept;
          row_value(true, vv, kept);
          if (kept) n_inrange++;
          t = tn;
          row++;
        }
        // At the end of the rows every lane closes bucket bidx; at a handoff only the lanes already in bidx + 1 have closed
        // it (their partials are committed, the other lanes keep their run of bidx for the segment loop).
        const bool done = row >= n_rows;
        if (done && !crossed) {
          va.fold(pt, NARROW);
          stage_lane<VK>(stage, staged, va.count != 0, va);
        }
        const bool filled = crossed || done;
        if (__any_sync(FULL, filled)) commit(filled);
        have_run = crossed || !done;
        run_idx = crossed ? bidx + 1 : bidx;
        pend_t = t;
        bk.valid = false;
        if (done) check_values();
      }
    }
  }

  // The warp walks its 32 pages SEGMENT by segment (a segment = rows of one page sharing (selected, bucket)), and for
  // GROUP BY bucket / tags it keeps the lanes aligned on the BUCKET: in every iteration only the lanes whose next selected
  // segment lies in the smallest pending bucket go ahead (the others keep their segment pending, at most an iteration
  // or two). Pages whose first row falls just before a bucket edge would otherwise run one segment ahead of their
  // neighbours for the whole page, no two lanes would ever finish a run for the same cell in the same iteration, and
  // every flush would degenerate into 32 contended atomics instead of one staged store per lane.
  const bool align = (P.width > 0 || EDGES) && !P.group_by_series;
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
            if (EDGES) {
              nb = edge_rows(P, bidx, rle_t0 + (uint64_t)row * rle_delta, rle_delta, rle_inv);
            } else {
              nb = q32 + (e_off < w_rem ? 1u : 0u);
              e_off = e_off + (uint64_t)nb * rle_delta - (uint64_t)P.width;
            }
          }
          if (bidx >= P.n_buckets) {
            report_error(P, TSKV_ERR_BUCKET_RANGE, page);
            seg_in = false;
            n_rows = row;
            pending = false;
          } else {
            seg_n = min(nb, rb1 - row);
            seg_b = bidx;
            if (P.width > 0 || EDGES) nb -= seg_n;
          }
        }
      } else {
        lim_lo = lim_hi = pend_t;
        seg_in = range_span(P, pend_t, lim_lo, lim_hi);
        if constexpr (TK == TK_GEN) seg_in = seg_in && !tcur.none;
        if (P.has_tomb) {  // decode_pages' tombstone handling (reader.rs:507-551) as two more segment attributes
          const uint4 tl = s_tomb[threadIdx.x];
          const bool dropped = tomb_span(P.tomb_ranges, P.n_tomb_global, pend_t, lim_lo, lim_hi) |
                               tomb_span(P.tomb_ranges + tl.x, tl.y, pend_t, lim_lo, lim_hi);
          seg_masked = tomb_span(P.tomb_ranges + tl.z, tl.w, pend_t, lim_lo, lim_hi);
          if (dropped) seg_in = false;
        }
        if (seg_in) {
          if (!(bk.valid && pend_t >= bk.lo && pend_t <= bk.hi) && !locate_bucket<EDGES>(P, pend_t, bk)) {
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
      if constexpr (M2)  // a run never changes cell: its shift is loaded once (pass-2 columns keep it at count_off)
        va.kmin = (int64_t)P.state[P.cols[qcol].count_off + group_base + bucket_cell<EDGES>(P, run_idx)];
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
          if constexpr (TK == TK_GEN) {  // only rows with a timestamp advance the cursor, never past the last row
            if (row < n_rows) {
              if ((row & 31) == 0) tcur.word = __ldg(tcur.bm + (row >> 5));
              if ((tcur.word >> (row & 31)) & 1) t = (int64_t)tcur.next();
            }
          } else {
            t = (int64_t)tcur.next();  // (past the last row this runs one value too far - harmless)
          }
          more = row < n_rows && (uint64_t)t - (uint64_t)lim_lo <= span;
        } while (more);
        pend_t = t;
        if (cursor_exhausted(tcur) && (TK == TK_GEN || row < n_rows)) {
          report_error(P, TSKV_ERR_BITSET_MISMATCH, P.time_page_of[page]);
          n_rows = row;
        }
      }
      check_values();
    }
  }
  if (!SEL && staged) {  // partials still parked in the staging area
    reduce_staged<VK, NS, M2>(P, stab, stage, staged);
    staged = 0;
  }
  // (only the lane that decodes the page's last rows walks on to the sentinel)
  if (VK == VK_GOR && have_item && n_rows != 0 && to_page_end && vcur_g.consumed_any() && !vcur_g.drain())  // float.rs:480-591
    report_error(P, TSKV_ERR_SHORT_BLOCK, page);
  ring_drain();  // nothing in flight when the next chunk reuses the rings
  if constexpr (M2) return;  // (pass 1 counted these rows)
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
// of the work; a warp repeatedly grabs one 32-item chunk of its bin from the bin's global counter and runs it through
// scan_chunk_seg, whatever the bin's time class.
#ifndef SCAN_MIN_BLOCKS
#define SCAN_MIN_BLOCKS 4
#endif
// 4 blocks of 4 warps per SM: 128 registers per thread. On sm_90a (ptxas -v) that keeps the variants without FIRST /
// LAST free of spills; the FIRST / LAST variants spill 4-146 bytes. A fifth block per SM would cap them at 96 registers
// and move the row loop's state into local memory.
__host__ __device__ constexpr int scan_min_blocks(int /*tk*/, bool /*sel*/) { return SCAN_MIN_BLOCKS; }
// staging-ring bytes one warp of the fused kernel needs: a value ring, and a time ring for simple8b timestamps (generic
// time pages are read from global memory)
__host__ __device__ constexpr uint32_t scan_ring_bytes_per_warp(int tk) {
  return tk == TK_S8B ? 2 * RING_BYTES_PER_WARP : RING_BYTES_PER_WARP;
}
// per-warp shared memory of the fused kernel: staging rings + the staged-flush area
__host__ __device__ constexpr uint32_t scan_warp_bytes(int tk) {
  return scan_ring_bytes_per_warp(tk) + flush_stage_bytes(flush_slots(tk));
}
// per-lane tombstone lists (tomb_lookup), after the warps' areas; allocated only when the page set has tombstones
constexpr uint32_t SCAN_TOMB_BYTES = SCAN_THREADS * sizeof(uint4);
// Narrow pages of a simple8b-value bin (ScanParams.page_narrow), per page set: none, some or all of them. NARROW_SOME
// kernels choose per chunk; NARROW_ALL kernels hold the narrow arithmetic only (a kernel that holds both row loops runs
// its narrow chunks ~1.5 % slower on C4: H100, see DESIGN.md §5).
enum { NARROW_NONE = 0, NARROW_SOME = 1, NARROW_ALL = 2 };
template <int TK, int VK, bool SEL, int NARROW, bool EDGES>
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
  // the bin's buckets (one per query column and narrow flag): groups of 32 items that never straddle two buckets
  uint32_t n_groups = 0;
  for (uint32_t k = bin * P.n_cols * WL_SUB; k < (bin + 1) * P.n_cols * WL_SUB; k++) n_groups += (__ldg(P.region_fill + k) + 31) >> 5;
  // pages cut at restart points: n_parts chunks per group of 32 pages (consecutive chunk numbers = the parts of one group)
  const uint32_t n_parts = (TK == TK_GEN || VK == VK_GEN || SEL) ? 1u : P.bin_parts[bin];
  const uint32_t part_rows = P.bin_part_rows[bin];
  const uint32_t n_chunks = n_groups * n_parts;
  for (;;) {
    uint32_t c = 0;
    if (lane == 0) c = atomicAdd(P.task_counter + bin, 1u);
    c = __shfl_sync(FULL, c, 0);
    if (c >= n_chunks) break;
    uint32_t group = n_parts > 1 ? c / n_parts : c;
    const uint32_t part = c - group * n_parts;
    uint32_t k = bin * P.n_cols * WL_SUB;
    asm("" : "+r"(k));  // computed here, per chunk: addresses hoisted out of the loop would hold registers of the row loops
    uint32_t fill = __ldg(P.region_fill + k);
    while (group >= (fill + 31) >> 5) {  // the bucket of the group, and the group's number inside it
      group -= (fill + 31) >> 5;
      fill = __ldg(P.region_fill + ++k);
    }
    const uint32_t region = __ldg(P.region_start + k);
    const uint32_t begin = region + (group << 5);
    const uint32_t end = min(begin + 32, region + fill);
    if constexpr (NARROW == NARROW_SOME) {
      // 32-bit arithmetic when all of the chunk's pages are narrow (a chunk holds one bucket: narrow or wide pages; the
      // vote also covers page sets without narrow flags in the work list)
      const uint32_t item = begin + lane;
      const bool narrow = __all_sync(FULL, item >= end || __ldg(P.page_narrow + __ldg(P.work_page + item)));
      if (narrow) scan_chunk_seg<TK, VK, SEL, true, EDGES>(P, begin, end, ring_base, s_tab, stage, s_tomb, part, n_parts, part_rows);
      else scan_chunk_seg<TK, VK, SEL, false, EDGES>(P, begin, end, ring_base, s_tab, stage, s_tomb, part, n_parts, part_rows);
    } else {
      scan_chunk_seg<TK, VK, SEL, NARROW == NARROW_ALL, EDGES>(P, begin, end, ring_base, s_tab, stage, s_tomb, part, n_parts, part_rows);
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

// Pass 2 of TSKV_AGG_M2: the fused kernel of bin `bin` once more, over the work-list regions of the M2 columns only
// (P.region_fill: pass 1's fills with every other column's set to 0, k_m2_prep), with the pass-2 column table (M2Col):
// count_off = the cells' shifts, sum_off / sumhi_off = sum(d) / sum(d^2), s_sum / s_hi in the shared-memory table. Narrow
// pages take the wide arithmetic. Own instantiations, so that the pass-1 kernels hold none of this code.
template <int TK, int VK, bool EDGES>
__global__ void __launch_bounds__(SCAN_THREADS, scan_min_blocks(TK, false)) k_scan_m2(const __grid_constant__ ScanParams P, int bin) {
  extern __shared__ __align__(16) uint64_t s_tab[];
  if (P.use_smem) {  // identities: +0.0
    for (uint32_t i = threadIdx.x; i < P.smem_words; i += SCAN_THREADS) s_tab[i] = 0;
    __syncthreads();
  }
  const uint32_t lane = threadIdx.x & 31;
  uint64_t *warp_area = s_tab + ((P.smem_words + 1) & ~1u) + (size_t)(threadIdx.x >> 5) * (scan_warp_bytes(TK) / 8);
  const uint32_t ring_base = (uint32_t)__cvta_generic_to_shared(warp_area);
  uint64_t *stage = warp_area + scan_ring_bytes_per_warp(TK) / 8;
  uint4 *s_tomb = reinterpret_cast<uint4 *>(s_tab + ((P.smem_words + 1) & ~1u) + (SCAN_THREADS / 32) * (scan_warp_bytes(TK) / 8));
  uint32_t n_groups = 0;
  for (uint32_t k = bin * P.n_cols * WL_SUB; k < (bin + 1) * P.n_cols * WL_SUB; k++) n_groups += (__ldg(P.region_fill + k) + 31) >> 5;
  const uint32_t n_parts = (TK == TK_GEN || VK == VK_GEN) ? 1u : P.bin_parts[bin];
  const uint32_t part_rows = P.bin_part_rows[bin];
  const uint32_t n_chunks = n_groups * n_parts;
  for (;;) {
    uint32_t c = 0;
    if (lane == 0) c = atomicAdd(P.task_counter + bin, 1u);
    c = __shfl_sync(FULL, c, 0);
    if (c >= n_chunks) break;
    uint32_t group = n_parts > 1 ? c / n_parts : c;
    const uint32_t part = c - group * n_parts;
    uint32_t k = bin * P.n_cols * WL_SUB;
    uint32_t fill = __ldg(P.region_fill + k);
    while (group >= (fill + 31) >> 5) {
      group -= (fill + 31) >> 5;
      fill = __ldg(P.region_fill + ++k);
    }
    const uint32_t region = __ldg(P.region_start + k);
    const uint32_t begin = region + (group << 5);
    const uint32_t end = min(begin + 32, region + fill);
    scan_chunk_seg<TK, VK, false, false, EDGES, true>(P, begin, end, ring_base, s_tab, stage, s_tomb, part, n_parts, part_rows);
  }
  if (P.use_smem) {  // merge this CTA's table into the global state, once
    __syncthreads();
    for (uint32_t c = 0; c < P.n_cols; c++) {
      const ColState cs = P.cols[c];
      if (!(cs.agg_mask & TSKV_AGG_M2)) continue;
      for (uint32_t i = threadIdx.x; i < (uint32_t)P.n_cells; i += SCAN_THREADS) {
        const uint64_t sd = s_tab[cs.s_sum + i], sd2 = s_tab[cs.s_hi + i];
        if (sd) atomicAdd(reinterpret_cast<double *>(P.state + cs.sum_off + i), __longlong_as_double((long long)sd));
        if (sd2) atomicAdd(reinterpret_cast<double *>(P.state + cs.sumhi_off + i), __longlong_as_double((long long)sd2));
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

// The scan's per-pass scratch ("aux" block): word offsets (8-byte words) of its parts.
constexpr uint32_t AUX_TASK_COUNTERS = 0;  // u32 ScanParams::task_counter[N_BINS]
constexpr uint32_t AUX_STATUS = 8;         // i32 ScanParams::status
constexpr uint32_t AUX_ERR_PAGE = 9;
constexpr uint32_t AUX_STATS = 10;         // ScanParams::stats[2]
constexpr uint32_t AUX_COUNTERS = 12;      // the reader counters (CTR_*)
constexpr uint32_t AUX_CRC_STATUS = AUX_COUNTERS + N_COUNTERS;  // i32: a page of k_verify_crc failed
constexpr uint32_t AUX_CRC_ERR_PAGE = AUX_CRC_STATUS + 1;
constexpr uint32_t AUX_WORDS = 32;
static_assert(N_BINS * 4 <= (AUX_STATUS - AUX_TASK_COUNTERS) * 8 && AUX_CRC_ERR_PAGE < AUX_WORDS, "scan aux block layout");

// Identities of the partial state; the same launch zeroes the scan's small per-pass scratch (the aux block, the
// work-list buckets' fill counts) so that a pass starts with ONE node instead of three memsets + a kernel.
__global__ void k_init_state(uint64_t *state, StateLayout L, unsigned long long *aux, uint32_t aux_words, uint32_t *zero32,
                             uint32_t n_zero32) {
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t k = i; k < aux_words; k += stride) aux[k] = 0;
  for (uint64_t k = i; k < n_zero32; k += stride) zero32[k] = 0;
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

// TSKV_AGG_M2 of one query column: state offsets (8-byte words) of its pass-1 count and f64 sum (the f64 sum of an F64
// column, the exported exact integer sum otherwise), and of its pass-2 arrays: the cells' shifts, sum(d) and sum(d^2).
struct M2Col {
  uint64_t count_off, sum_off, shift_off, sd_off, sd2_off;
};

// Between the passes: shift[cell] = pass-1 sum / count (0 for an empty cell) of every M2 column (blockIdx.y); block
// (0, 0) also writes pass 2's bucket fills (pass 1's, with the buckets of columns without M2 set to 0: pass 2 launches
// over the M2 columns' regions only) and zeroes pass 2's task counters.
__global__ void k_m2_prep(uint64_t *state, const M2Col *m2, uint64_t n_cells, const uint32_t *fill, uint32_t *fill2,
                          uint32_t n_buckets, const ColState *cols2, uint32_t n_cols, uint32_t *task_counter) {
  const M2Col mc = m2[blockIdx.y];
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_cells; i += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t n = state[mc.count_off + i];
    const double s = __longlong_as_double((long long)state[mc.sum_off + i]);
    state[mc.shift_off + i] = (uint64_t)__double_as_longlong(n ? s / (double)n : 0.0);
  }
  if (blockIdx.x == 0 && blockIdx.y == 0) {
    for (uint32_t k = threadIdx.x; k < n_buckets; k += blockDim.x)
      fill2[k] = (cols2[(k / WL_SUB) % n_cols].agg_mask & TSKV_AGG_M2) ? fill[k] : 0u;
    for (uint32_t b = threadIdx.x; b < N_BINS; b += blockDim.x) task_counter[b] = 0;
  }
}

// Multi-GPU, after k_merge_gathered: M2 of every M2 column (blockIdx.y) and cell from the gathered ranks' (count n_r,
// shift c_r, sum(d), sum(d^2)), each rank's d taken around its own shift: M2_r = sum(d^2) - sum(d)^2 / n_r, and the
// rank's mean relative to the shift c of the first rank holding the cell, mu_r = (c_r - c) + sum(d) / n_r (close means:
// the difference of the shifts is exact). Chan's merge M2 = sum M2_r + sum n_r (mu_r - mu)^2, mu = sum n_r mu_r / n.
// (Relative means keep the digits that means near 2^63 as f64 would lose.) Writes sum(d) = 0 and sum(d^2) = M2, which
// k_finalize turns into M2 again.
__global__ void k_merge_m2(uint64_t *state, const M2Col *m2, uint64_t n_cells, const uint64_t *gathered, uint32_t n_ranks,
                           uint64_t exch_words) {
  const M2Col mc = m2[blockIdx.y];
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_cells; i += (uint64_t)gridDim.x * blockDim.x) {
    auto at = [&](uint32_t r, uint64_t off) { return gathered[r * exch_words + off + i]; };
    auto f64 = [&](uint32_t r, uint64_t off) { return __longlong_as_double((long long)at(r, off)); };
    uint64_t n = 0;
    double c = 0.0, mu_sum = 0.0;
    bool have_c = false;
    for (uint32_t r = 0; r < n_ranks; r++) {
      const uint64_t nr = at(r, mc.count_off);
      if (!nr) continue;
      if (!have_c) { c = f64(r, mc.shift_off); have_c = true; }
      n += nr;
      mu_sum += (f64(r, mc.shift_off) - c) * (double)nr + f64(r, mc.sd_off);
    }
    double acc = 0.0;
    if (n) {
      const double mu = mu_sum / (double)n;
      for (uint32_t r = 0; r < n_ranks; r++) {
        const uint64_t nr = at(r, mc.count_off);
        if (!nr) continue;
        const double sd = f64(r, mc.sd_off), sd2 = f64(r, mc.sd2_off);
        const double dm = (f64(r, mc.shift_off) - c) + sd / (double)nr - mu;
        acc += (sd2 - sd * sd / (double)nr) + (double)nr * dm * dm;
      }
    }
    state[mc.sd_off + i] = 0;
    state[mc.sd2_off + i] = (uint64_t)__double_as_longlong(acc);
  }
}

// ---- column pairs (tskv_query.n_pairs): covariance / correlation state ---------------------------------------------
// One pair's state is PAIR_WORDS sections of n_cells words from `off` on (PairSec), right after the M2 sections so that
// the exchange region holds them. Pass 1 (k_scan_pair<false>) sums the paired rows' n, x and y and keeps the order keys
// of their smallest and largest f64 x and y (pair_ukey; a min is kept as ~key so that every section starts at 0 and
// grows with atomicMax); k_pair_prep writes the shifts sum / n; pass 2 sums dx, dy, dx dy, dx^2 and dy^2 around them.
enum PairSec { PS_N = 0, PS_SX, PS_SY, PS_XMIN, PS_XMAX, PS_YMIN, PS_YMAX, PS_SHX, PS_SHY, PS_DX, PS_DY, PS_DXY, PS_DX2,
               PS_DY2, PAIR_WORDS };
struct PairCol {
  uint64_t off;          // first word of the pair's sections
  uint32_t qx, qy;       // the operands' columns in the scan's column table (work-list buckets: x's)
  uint16_t x_id, y_id;
  uint8_t x_pt, y_pt;
  uint8_t pad[2];
};

__device__ __forceinline__ double pair_f64(uint64_t v, uint8_t pt) {  // the operand as f64, as DataFusion converts it
  return pt == TSKV_PT_F64 ? __longlong_as_double((long long)v) : pt == TSKV_PT_I64 ? (double)(int64_t)v : (double)v;
}
__device__ __forceinline__ unsigned long long pair_ukey(double d) {  // unsigned order key of an f64 value
  return (unsigned long long)okey((uint64_t)__double_as_longlong(d), TSKV_PT_F64) ^ 0x8000000000000000ull;
}

// The sums of one run of paired rows (one cell) of one lane, flushed with one atomic per quantity.
struct PairAcc {
  uint64_t n;
  double a, b, c, d, e;                      // pass 1: sum x, sum y; pass 2: sum dx, sum dy, sum dx dy, sum dx^2, sum dy^2
  unsigned long long xmin, xmax, ymin, ymax;  // pass 1: ~key / key of the extreme x and y
  double shx, shy;                           // pass 2: the cell's shifts
};
template <bool PASS2>
__device__ __forceinline__ void pair_start(const ScanParams &P, const PairCol &pc, uint64_t cell, PairAcc &r) {
  r.n = 0; r.a = r.b = r.c = r.d = r.e = 0.0;
  r.xmin = r.xmax = r.ymin = r.ymax = 0;
  if (PASS2) {
    r.shx = __longlong_as_double((long long)P.state[pc.off + PS_SHX * P.n_cells + cell]);
    r.shy = __longlong_as_double((long long)P.state[pc.off + PS_SHY * P.n_cells + cell]);
  }
}
template <bool PASS2>
__device__ __forceinline__ void pair_add(PairAcc &r, double x, double y) {
  r.n++;
  if (PASS2) {
    const double dx = x - r.shx, dy = y - r.shy;
    r.a += dx; r.b += dy; r.c += dx * dy; r.d += dx * dx; r.e += dy * dy;
  } else {
    r.a += x; r.b += y;
    const unsigned long long kx = pair_ukey(x), ky = pair_ukey(y);
    r.xmin = max(r.xmin, ~kx); r.xmax = max(r.xmax, kx);
    r.ymin = max(r.ymin, ~ky); r.ymax = max(r.ymax, ky);
  }
}
template <bool PASS2>
__device__ __forceinline__ void pair_flush(const ScanParams &P, const PairCol &pc, uint64_t cell, const PairAcc &r) {
  if (!r.n) return;
  uint64_t *s = P.state + pc.off + cell;
  auto f = [&](int sec, double v) { atomicAdd(reinterpret_cast<double *>(s + sec * P.n_cells), v); };
  auto m = [&](int sec, unsigned long long v) { atomicMax(reinterpret_cast<unsigned long long *>(s + sec * P.n_cells), v); };
  if (PASS2) {
    f(PS_DX, r.a); f(PS_DY, r.b); f(PS_DXY, r.c); f(PS_DX2, r.d); f(PS_DY2, r.e);
  } else {
    atomicAdd(reinterpret_cast<unsigned long long *>(s + PS_N * P.n_cells), (unsigned long long)r.n);
    f(PS_SX, r.a); f(PS_SY, r.b);
    m(PS_XMIN, r.xmin); m(PS_XMAX, r.xmax); m(PS_YMIN, r.ymin); m(PS_YMAX, r.ymax);
  }
}

// The row selection of the column pairs and the medians, as scan_chunk_seg selects: the keep bit of row r, the time
// ranges, the row-drop tombstones (global, and the series' in ta.x / ta.y) and the operands' column tombstones (ta.z /
// ta.w, tb.z / tb.w), then the bucket of timestamp t (bk caches the last one). Sets the row's cell when it is selected.
template <bool EDGES>
__device__ __forceinline__ bool select_row(const ScanParams &P, const uint32_t *keepw, uint32_t r, int64_t t, const uint4 &ta,
                                           const uint4 &tb, uint64_t group_base, BucketState &bk, uint64_t &cell) {
  if (keepw && !((__ldg(keepw + (r >> 5)) >> (r & 31)) & 1)) return false;
  int64_t lo, hi;
  if (!range_span(P, t, lo, hi)) return false;
  if (P.has_tomb && (tomb_span(P.tomb_ranges, P.n_tomb_global, t, lo, hi) | tomb_span(P.tomb_ranges + ta.x, ta.y, t, lo, hi) |
                     tomb_span(P.tomb_ranges + ta.z, ta.w, t, lo, hi) | tomb_span(P.tomb_ranges + tb.z, tb.w, t, lo, hi)))
    return false;
  if (!(bk.valid && t >= bk.lo && t <= bk.hi) && !locate_bucket<EDGES>(P, t, bk)) { bk.valid = false; return false; }  // (pass 1 reports it)
  cell = group_base + bucket_cell<EDGES>(P, bk.idx);
  return true;
}

// One x page of a pair (work item `item` of x's buckets) and the y page of the same column group, decoded in lock-step
// with the group's time page row by row; a row counts when scan_chunk_seg would select it (valid timestamp, keep bit,
// time ranges, row-drop tombstones) and both x and y hold a value that no column tombstone masks. The y page is found
// once per item in the group's descriptors. Decode errors of the three pages are pass 1's to report (every operand is a
// column of the scan): the lane stops at the first.
template <bool PASS2, bool EDGES>
__device__ __forceinline__ void pair_page(const ScanParams &P, const PairCol &pc, uint64_t n_descs, uint32_t item) {
  const uint32_t page = P.work_page[item], slot = P.work_slot[item];
  const tskv_page_desc xd = P.descs[page];
  const uint32_t tpage = P.time_page_of[page];
  const tskv_page_desc td = P.descs[tpage];
  uint32_t ypage = FULL;
  for (uint64_t p = tpage + 1; p < n_descs && P.descs[p].phys_type != TSKV_PT_TIME; p++)
    if (P.descs[p].column_id == pc.y_id) { ypage = (uint32_t)p; break; }
  if (ypage == FULL) return;  // the group holds no y: NULL for every row (the reference null-fills it)
  const tskv_page_desc yd = P.descs[ypage];
  if (yd.phys_type != pc.y_pt || kind_status(xd.reserved) != TSKV_OK || kind_status(yd.reserved) != TSKV_OK ||
      kind_status(td.reserved) != TSKV_OK || td.reserved == DK_ALLNULL || xd.reserved == DK_ALLNULL || yd.reserved == DK_ALLNULL)
    return;
  PageView tpv, xpv, ypv;
  tpv.open(P.arena, td);
  xpv.open(P.arena, xd);
  ypv.open(P.arena, yd);
  BitCursor tb, xb, yb;
  tb.init(tpv.bitset);
  xb.init(xpv.bitset);
  yb.init(ypv.bitset);
  DeltaCursor<-1> tc;
  AnyCursor<> xc, yc;
  if (tc.open(tpv, td.reserved) != TSKV_OK || xc.open(xpv, xd.reserved) != TSKV_OK || yc.open(ypv, yd.reserved) != TSKV_OK) return;
  uint4 tx = make_uint4(0, 0, 0, 0), ty = tx;
  if (P.has_tomb) {
    tx = tomb_lookup(P, xd.series_id, pc.x_id);
    ty = tomb_lookup(P, xd.series_id, pc.y_id);
  }
  const uint32_t *keepw = P.row_keep ? P.row_keep + P.keep_off[tpage] : nullptr;
  const uint64_t group_base = group_cell_base<EDGES>(P, slot);
  BucketState bk; bk.valid = false; bk.floor_regime = false; bk.lo = 0; bk.hi = 0; bk.idx = 0;
  PairAcc acc;
  uint64_t run_cell = 0;
  bool have_run = false;
  int64_t t = 0;
  const uint32_t n_rows = xd.num_values;
  for (uint32_t r = 0; r < n_rows; r++) {
    const bool tv = tb.next(r), xv = xb.next(r), yv = yb.next(r);
    uint64_t xr = 0, yr = 0;
    if (tv) { t = (int64_t)tc.next(); if (tc.exhausted) break; }
    else if (r == 0) tc.skip_first_if_s8b_sc();
    if (xv) { xr = xc.next(); if (xc.failed()) break; }
    else if (r == 0 && !xc.is_gorilla) xc.d.skip_first_if_s8b_sc();
    if (yv) { yr = yc.next(); if (yc.failed()) break; }
    else if (r == 0 && !yc.is_gorilla) yc.d.skip_first_if_s8b_sc();
    uint64_t cell;
    if (!(tv && xv && yv) || !select_row<EDGES>(P, keepw, r, t, tx, ty, group_base, bk, cell)) continue;
    if (!have_run || cell != run_cell) {
      if (have_run) pair_flush<PASS2>(P, pc, run_cell, acc);
      pair_start<PASS2>(P, pc, cell, acc);
      run_cell = cell;
      have_run = true;
    }
    pair_add<PASS2>(acc, pair_f64(xr, pc.x_pt), pair_f64(yr, pc.y_pt));
  }
  if (have_run) pair_flush<PASS2>(P, pc, run_cell, acc);
}

// Pass 1 / pass 2 of the column pairs (blockIdx.y: the pair): one lane per work item of the x operand's buckets (every
// bin, wide and narrow), the same items pass 1 of the column scan read. Own kernels with their own arguments, so that the
// fused kernels and ScanParams stay as they are.
template <bool PASS2, bool EDGES>
__global__ void __launch_bounds__(128) k_scan_pair(const __grid_constant__ ScanParams P, const PairCol *pairs, uint64_t n_descs) {
  const PairCol pc = pairs[blockIdx.y];
  const uint32_t stride = gridDim.x * blockDim.x, t0 = blockIdx.x * blockDim.x + threadIdx.x;
  for (uint32_t k = pc.qx * WL_SUB; k < N_BINS * P.n_cols * WL_SUB; k += P.n_cols * WL_SUB)
    for (uint32_t sub = 0; sub < WL_SUB; sub++) {
      const uint32_t start = __ldg(P.region_start + k + sub), fill = __ldg(P.region_fill + k + sub);
      for (uint32_t i = t0; i < fill; i += stride) pair_page<PASS2, EDGES>(P, pc, n_descs, start + i);
    }
}

// Between the pair passes: the shifts sum x / n and sum y / n of every cell (0 for an empty cell).
__global__ void k_pair_prep(uint64_t *state, const PairCol *pairs, uint64_t n_cells) {
  const PairCol pc = pairs[blockIdx.y];
  uint64_t *s = state + pc.off;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_cells; i += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t n = s[PS_N * n_cells + i];
    const double sx = __longlong_as_double((long long)s[PS_SX * n_cells + i]), sy = __longlong_as_double((long long)s[PS_SY * n_cells + i]);
    s[PS_SHX * n_cells + i] = (uint64_t)__double_as_longlong(n ? sx / (double)n : 0.0);
    s[PS_SHY * n_cells + i] = (uint64_t)__double_as_longlong(n ? sy / (double)n : 0.0);
  }
}

// Multi-GPU, after k_merge_gathered: every pair's cells from the gathered ranks' sections. Each rank's co-moments are
// taken around its own shifts; its means relative to the shifts of the first rank holding the cell (as k_merge_m2) enter
// Chan's formulas C = sum C_r + sum n_r (mx_r - mx)(my_r - my), M2 = sum M2_r + sum n_r (m_r - m)^2. Writes n, the extreme
// keys, sum dx = sum dy = 0 and sum dx dy = C, sum dx^2 = M2x, sum dy^2 = M2y, which k_finalize_pairs reads unchanged.
__global__ void k_merge_pairs(uint64_t *state, const PairCol *pairs, uint64_t n_cells, const uint64_t *gathered, uint32_t n_ranks,
                              uint64_t exch_words) {
  const PairCol pc = pairs[blockIdx.y];
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_cells; i += (uint64_t)gridDim.x * blockDim.x) {
    auto at = [&](uint32_t r, int sec) { return gathered[r * exch_words + pc.off + sec * n_cells + i]; };
    auto f64 = [&](uint32_t r, int sec) { return __longlong_as_double((long long)at(r, sec)); };
    uint64_t n = 0;
    unsigned long long km[4] = {0, 0, 0, 0};
    double cx = 0.0, cy = 0.0, mx_sum = 0.0, my_sum = 0.0;
    bool have_c = false;
    for (uint32_t r = 0; r < n_ranks; r++) {
      for (int q = 0; q < 4; q++) km[q] = max(km[q], (unsigned long long)at(r, PS_XMIN + q));
      const uint64_t nr = at(r, PS_N);
      if (!nr) continue;
      if (!have_c) { cx = f64(r, PS_SHX); cy = f64(r, PS_SHY); have_c = true; }
      n += nr;
      mx_sum += (f64(r, PS_SHX) - cx) * (double)nr + f64(r, PS_DX);
      my_sum += (f64(r, PS_SHY) - cy) * (double)nr + f64(r, PS_DY);
    }
    double c = 0.0, m2x = 0.0, m2y = 0.0;
    if (n) {
      const double mx = mx_sum / (double)n, my = my_sum / (double)n;
      for (uint32_t r = 0; r < n_ranks; r++) {
        const uint64_t nr = at(r, PS_N);
        if (!nr) continue;
        const double sdx = f64(r, PS_DX), sdy = f64(r, PS_DY), inv = 1.0 / (double)nr;
        const double dmx = (f64(r, PS_SHX) - cx) + sdx * inv - mx, dmy = (f64(r, PS_SHY) - cy) + sdy * inv - my;
        c += (f64(r, PS_DXY) - sdx * sdy * inv) + (double)nr * dmx * dmy;
        m2x += (f64(r, PS_DX2) - sdx * sdx * inv) + (double)nr * dmx * dmx;
        m2y += (f64(r, PS_DY2) - sdy * sdy * inv) + (double)nr * dmy * dmy;
      }
    }
    uint64_t *s = state + pc.off + i;
    s[PS_N * n_cells] = n;
    for (int q = 0; q < 4; q++) s[(PS_XMIN + q) * n_cells] = km[q];
    s[PS_DX * n_cells] = s[PS_DY * n_cells] = 0;
    s[PS_DXY * n_cells] = (uint64_t)__double_as_longlong(c);
    s[PS_DX2 * n_cells] = (uint64_t)__double_as_longlong(m2x);
    s[PS_DY2 * n_cells] = (uint64_t)__double_as_longlong(m2y);
  }
}

// M2 of one operand from its pass-2 sums: the corrected two-pass formula clamped at 0, and exactly 0 when every paired
// value is the same finite number (the shift's rounding residue would otherwise make corr of a constant column noise).
__device__ __forceinline__ double pair_m2(double sd, double sd2, uint64_t n, unsigned long long nkmin, unsigned long long kmax) {
  if (~nkmin == kmax) {
    const uint64_t bits = (uint64_t)okey_inv((int64_t)(kmax ^ 0x8000000000000000ull), TSKV_PT_F64);
    if (isfinite(__longlong_as_double((long long)bits))) return 0.0;
  }
  const double m2 = sd2 - sd * sd / (double)n;
  return m2 < 0.0 ? 0.0 : m2;
}

// The four outputs of every pair (blockIdx.y = 4 * pair + j; output column out0 + blockIdx.y): j = 0 n (always valid),
// 1 C, 2 M2x, 3 M2y (valid iff n >= 1).
__global__ void k_finalize_pairs(const uint64_t *state, const PairCol *pairs, uint32_t out0, uint64_t n_cells, uint64_t bitmap_stride,
                                 uint64_t *values, uint8_t *validity) {
  const PairCol pc = pairs[blockIdx.y >> 2];
  const uint32_t j = blockIdx.y & 3;
  const uint64_t cell = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  bool valid = false;
  if (cell < n_cells) {
    const uint64_t *s = state + pc.off + cell;
    auto f64 = [&](int sec) { return __longlong_as_double((long long)s[sec * n_cells]); };
    const uint64_t n = s[PS_N * n_cells];
    double v = 0.0;
    valid = j == 0 || n > 0;
    if (j != 0 && n) {
      if (j == 1) v = f64(PS_DXY) - f64(PS_DX) * f64(PS_DY) / (double)n;
      else if (j == 2) v = pair_m2(f64(PS_DX), f64(PS_DX2), n, s[PS_XMIN * n_cells], s[PS_XMAX * n_cells]);
      else v = pair_m2(f64(PS_DY), f64(PS_DY2), n, s[PS_YMIN * n_cells], s[PS_YMAX * n_cells]);
    }
    values[(uint64_t)(out0 + blockIdx.y) * n_cells + cell] = j == 0 ? n : (uint64_t)__double_as_longlong(v);
  }
  const uint32_t bits = __ballot_sync(FULL, valid);
  if ((threadIdx.x & 31) == 0 && (cell >> 3) < bitmap_stride)
    *reinterpret_cast<uint32_t *>(validity + (uint64_t)(out0 + blockIdx.y) * bitmap_stride + (cell >> 3)) = bits;
}

// ---- medians (TSKV_QUERY_N_MEDIANS): exact selection over the cells' unsigned order keys ------------------------------
// Pass 1 (the fused scan) leaves every cell's n, smallest and largest key in the operand's COUNT / MIN / MAX sections.
// k_median_prep sets each cell's targets, ranks (n - 1) / 2 and n / 2, under the common leading bits of its two
// extremes. Every selection pass (k_scan_median, k_merge_median_rows for merged rows) counts the keys under a cell's
// prefix by their next 8-bit digit; k_median_step finds the digits that hold the ranks and extends the prefix. Once the
// two ranks of an even cell part, the lower one is the largest key under its prefix and the upper one the smallest
// under its own: one more pass takes both with atomicMax / atomicMin. 8 passes resolve any cell.
// A median's state is MEDIAN_WORDS sections of n_cells words from `off` on (MedianSec) and its histograms are
// MEDIAN_BINS u32 per cell from hist_off on; the count of unresolved cells follows every median's sections.
enum MedianSec { MS_MODE = 0, MS_BITS, MS_PLO, MS_PHI, MS_RLO, MS_RHI, MS_LO, MS_HI, MEDIAN_WORDS };
enum MedianMode { MM_DONE = 0, MM_HIST, MM_EXTREME };
constexpr uint32_t MEDIAN_BINS = 256;
constexpr int MEDIAN_PASSES = 8;  // 64 key bits / 8 per pass (a pass that parts the ranks leaves the extremes pass a digit)
struct MedianCol {
  uint64_t count_off, min_off, max_off;  // the operand's COUNT and MIN / MAX key sections in the scan state
  uint64_t off, hist_off;                // the median's sections in the median state, its histograms
  uint32_t qcol;                         // the operand's column in the scan's column table (its work-list buckets)
  uint16_t column_id;
  uint8_t phys_type;
  uint8_t pad;
};
// The pointers every median kernel takes: the median state, the histograms and the count of unresolved cells.
struct MedianArgs {
  uint64_t *state;
  uint32_t *hist;
  unsigned long long *unresolved;
};

__device__ __forceinline__ uint64_t median_ukey(uint64_t v, uint8_t pt) { return (uint64_t)okey(v, pt) ^ 0x8000000000000000ull; }
__device__ __forceinline__ bool median_under(uint64_t u, uint64_t prefix, uint32_t bits) {  // u has the prefix's leading bits
  return bits == 0 || ((u ^ prefix) >> (64 - bits)) == 0;
}
__device__ __forceinline__ uint32_t median_digit_shift(uint32_t bits) { return 64 - bits > 8 ? 56 - bits : 0; }
__device__ __forceinline__ uint32_t median_digit(uint64_t u, uint32_t bits) {  // the (up to) 8 bits after the prefix
  return (uint32_t)(u >> median_digit_shift(bits)) & ((1u << (64 - bits > 8 ? 8 : 64 - bits)) - 1);
}

// One lane's run of rows in one cell: the cell's selection state, and the pending histogram run of equal digits or the
// extremes under the two prefixes.
struct MedianRun {
  uint64_t cell, plo, phi, xlo, xhi;
  uint32_t mode, bits, digit, n;
  bool have_lo, have_hi;
};
__device__ __forceinline__ void median_flush(const MedianCol &mc, const MedianArgs &A, uint64_t n_cells, MedianRun &r) {
  if (r.mode == MM_HIST && r.n) atomicAdd(A.hist + mc.hist_off + r.cell * MEDIAN_BINS + r.digit, r.n);
  if (r.have_lo) atomicMax(reinterpret_cast<unsigned long long *>(A.state + mc.off + MS_LO * n_cells + r.cell), (unsigned long long)r.xlo);
  if (r.have_hi) atomicMin(reinterpret_cast<unsigned long long *>(A.state + mc.off + MS_HI * n_cells + r.cell), (unsigned long long)r.xhi);
  r.n = 0;
  r.have_lo = r.have_hi = false;
}
__device__ __forceinline__ void median_open(const MedianCol &mc, const MedianArgs &A, uint64_t n_cells, uint64_t cell, MedianRun &r) {
  const uint64_t *s = A.state + mc.off + cell;
  r.cell = cell;
  r.mode = (uint32_t)s[MS_MODE * n_cells];
  r.bits = (uint32_t)s[MS_BITS * n_cells];
  r.plo = s[MS_PLO * n_cells];
  r.phi = s[MS_PHI * n_cells];
  r.n = 0;
  r.have_lo = r.have_hi = false;
}
__device__ __forceinline__ void median_add(const MedianCol &mc, const MedianArgs &A, uint64_t n_cells, MedianRun &r, uint64_t u) {
  if (r.mode == MM_HIST) {
    if (!median_under(u, r.plo, r.bits)) return;
    const uint32_t d = median_digit(u, r.bits);
    if (r.n && d != r.digit) median_flush(mc, A, n_cells, r);
    r.digit = d;
    r.n++;
  } else if (r.mode == MM_EXTREME) {
    if (median_under(u, r.plo, r.bits)) { r.xlo = r.have_lo ? max(r.xlo, u) : u; r.have_lo = true; }
    if (median_under(u, r.phi, r.bits)) { r.xhi = r.have_hi ? min(r.xhi, u) : u; r.have_hi = true; }
  }
}

// One page of a median's operand (work item `item` of its buckets), decoded with its group's time page row by row and
// selected as the column pairs select (select_row). Decode errors are pass 1's to report: the lane stops at the first.
template <bool EDGES>
__device__ __forceinline__ void median_page(const ScanParams &P, const MedianCol &mc, const MedianArgs &A, uint32_t item) {
  const uint32_t page = P.work_page[item], slot = P.work_slot[item];
  const tskv_page_desc vd = P.descs[page];
  const uint32_t tpage = P.time_page_of[page];
  const tskv_page_desc td = P.descs[tpage];
  if (vd.phys_type != mc.phys_type || kind_status(vd.reserved) != TSKV_OK || kind_status(td.reserved) != TSKV_OK ||
      td.reserved == DK_ALLNULL || vd.reserved == DK_ALLNULL)
    return;
  PageView tpv, vpv;
  tpv.open(P.arena, td);
  vpv.open(P.arena, vd);
  BitCursor tb, vb;
  tb.init(tpv.bitset);
  vb.init(vpv.bitset);
  DeltaCursor<-1> tc;
  AnyCursor<> vc;
  if (tc.open(tpv, td.reserved) != TSKV_OK || vc.open(vpv, vd.reserved) != TSKV_OK) return;
  const uint4 none = make_uint4(0, 0, 0, 0);
  const uint4 tv4 = P.has_tomb ? tomb_lookup(P, vd.series_id, mc.column_id) : none;
  const uint32_t *keepw = P.row_keep ? P.row_keep + P.keep_off[tpage] : nullptr;
  const uint64_t group_base = group_cell_base<EDGES>(P, slot);
  BucketState bk; bk.valid = false; bk.floor_regime = false; bk.lo = 0; bk.hi = 0; bk.idx = 0;
  MedianRun run;
  run.mode = MM_DONE;
  run.cell = ~0ull;
  run.n = 0;
  run.have_lo = run.have_hi = false;
  int64_t t = 0;
  const uint32_t n_rows = vd.num_values;
  for (uint32_t r = 0; r < n_rows; r++) {
    const bool tv = tb.next(r), vv = vb.next(r);
    uint64_t v = 0;
    if (tv) { t = (int64_t)tc.next(); if (tc.exhausted) break; }
    else if (r == 0) tc.skip_first_if_s8b_sc();
    if (vv) { v = vc.next(); if (vc.failed()) break; }
    else if (r == 0 && !vc.is_gorilla) vc.d.skip_first_if_s8b_sc();
    uint64_t cell;
    if (!(tv && vv) || !select_row<EDGES>(P, keepw, r, t, tv4, none, group_base, bk, cell)) continue;
    if (cell != run.cell) {
      median_flush(mc, A, P.n_cells, run);
      median_open(mc, A, P.n_cells, cell, run);
    }
    median_add(mc, A, P.n_cells, run, median_ukey(v, mc.phys_type));
  }
  median_flush(mc, A, P.n_cells, run);
}

// One selection pass of the medians (blockIdx.y: the median): one lane per work item of the operand's buckets (every
// bin, wide and narrow), the items pass 1 read. Returns at once when every cell is resolved.
template <bool EDGES>
__global__ void __launch_bounds__(128) k_scan_median(const __grid_constant__ ScanParams P, const MedianCol *meds, const MedianArgs A) {
  if (*(volatile unsigned long long *)A.unresolved == 0) return;
  const MedianCol mc = meds[blockIdx.y];
  const uint32_t stride = gridDim.x * blockDim.x, t0 = blockIdx.x * blockDim.x + threadIdx.x;
  for (uint32_t k = mc.qcol * WL_SUB; k < N_BINS * P.n_cols * WL_SUB; k += P.n_cols * WL_SUB)
    for (uint32_t sub = 0; sub < WL_SUB; sub++) {
      const uint32_t start = __ldg(P.region_start + k + sub), fill = __ldg(P.region_fill + k + sub);
      for (uint32_t i = t0; i < fill; i += stride) median_page<EDGES>(P, mc, A, start + i);
    }
}

// After pass 1: every cell's targets. A cell with no value is done (NULL); one whose extremes are equal is done with
// that key; any other starts its histogram passes under the common leading bits of its extremes.
__global__ void k_median_prep(const uint64_t *state, const MedianCol *meds, const MedianArgs A, uint64_t n_cells) {
  const MedianCol mc = meds[blockIdx.y];
  uint64_t *s = A.state + mc.off;
  unsigned open = 0;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_cells; i += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t n = state[mc.count_off + i];
    const uint64_t kmin = state[mc.min_off + i] ^ 0x8000000000000000ull, kmax = state[mc.max_off + i] ^ 0x8000000000000000ull;
    const bool hist = n > 1 && kmin != kmax;
    const uint32_t bits = hist ? (uint32_t)__clzll((long long)(kmin ^ kmax)) : 64;
    const uint64_t prefix = bits == 0 ? 0 : kmin & (~0ull << (64 - bits));
    s[MS_MODE * n_cells + i] = hist ? MM_HIST : MM_DONE;
    s[MS_BITS * n_cells + i] = bits;
    s[MS_PLO * n_cells + i] = s[MS_PHI * n_cells + i] = prefix;
    s[MS_RLO * n_cells + i] = n ? (n - 1) / 2 : 0;
    s[MS_RHI * n_cells + i] = n / 2;
    s[MS_LO * n_cells + i] = s[MS_HI * n_cells + i] = kmin;
    open += hist;
  }
  open = __reduce_add_sync(FULL, open);
  if ((threadIdx.x & 31) == 0 && open) atomicAdd(A.unresolved, (unsigned long long)open);
}

// After a selection pass: a warp per cell. A histogram cell (lane l holds bins 8 l .. 8 l + 7) finds the digits that
// hold its two ranks, clears its bins and extends its prefixes; it is done when the key is complete, and goes to the
// extremes pass when the ranks part. An extremes cell is done (the pass left its keys in MS_LO / MS_HI).
__global__ void __launch_bounds__(256) k_median_step(const MedianCol *meds, const MedianArgs A, uint64_t n_cells) {
  if (*(volatile unsigned long long *)A.unresolved == 0) return;
  const MedianCol mc = meds[blockIdx.y];
  uint64_t *s = A.state + mc.off;
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t warps = (uint64_t)gridDim.x * (blockDim.x >> 5);
  for (uint64_t i = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n_cells; i += warps) {
    const uint64_t mode = s[MS_MODE * n_cells + i];
    if (mode == MM_DONE) continue;
    if (mode == MM_EXTREME) {
      if (lane == 0) {
        s[MS_MODE * n_cells + i] = MM_DONE;
        atomicAdd(A.unresolved, ~0ull);
      }
      continue;
    }
    uint4 *h = reinterpret_cast<uint4 *>(A.hist + mc.hist_off + i * MEDIAN_BINS) + 2 * lane;
    const uint4 a = h[0], b = h[1];
    h[0] = h[1] = make_uint4(0, 0, 0, 0);
    const uint32_t c[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
    uint64_t sum = 0;
#pragma unroll
    for (int k = 0; k < 8; k++) sum += c[k];
    uint64_t incl = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint64_t v = ((uint64_t)__shfl_up_sync(FULL, (uint32_t)(incl >> 32), o) << 32) | __shfl_up_sync(FULL, (uint32_t)incl, o);
      if (lane >= (uint32_t)o) incl += v;
    }
    const uint64_t excl = incl - sum;
    // the digit holding rank r and r's rank among the keys of that digit (found = false: the pass counted fewer keys
    // than pass 1, which only a decode error that pass 1 reports can cause)
    auto find = [&](uint64_t r, uint32_t &d, uint64_t &rest) {
      const uint32_t owner = __ballot_sync(FULL, excl <= r && r < incl);
      if (!owner) return false;
      const int src = __ffs(owner) - 1;
      uint32_t dd = 0;
      uint64_t rr = r - excl;
      if ((int)lane == src)
        for (int k = 0; k < 8; k++) {
          if (rr < c[k]) { dd = 8 * lane + k; break; }
          rr -= c[k];
        }
      d = __shfl_sync(FULL, dd, src);
      rest = shfl_u64(rr, src);
      return true;
    };
    uint32_t dlo = 0, dhi = 0;
    uint64_t qlo = 0, qhi = 0;
    const bool found_lo = find(s[MS_RLO * n_cells + i], dlo, qlo);
    const bool found_hi = find(s[MS_RHI * n_cells + i], dhi, qhi);
    if (lane == 0) {
      const uint32_t bits = (uint32_t)s[MS_BITS * n_cells + i];
      const uint32_t sh = median_digit_shift(bits), nb = 64 - sh;
      const uint64_t plo = s[MS_PLO * n_cells + i] | ((uint64_t)dlo << sh), phi = s[MS_PLO * n_cells + i] | ((uint64_t)dhi << sh);
      s[MS_BITS * n_cells + i] = nb;
      s[MS_PLO * n_cells + i] = plo;
      s[MS_PHI * n_cells + i] = phi;
      s[MS_RLO * n_cells + i] = qlo;
      s[MS_RHI * n_cells + i] = qhi;
      if (nb == 64 || !found_lo || !found_hi) {
        s[MS_LO * n_cells + i] = plo;
        s[MS_HI * n_cells + i] = phi;
        s[MS_MODE * n_cells + i] = MM_DONE;
        atomicAdd(A.unresolved, ~0ull);
      } else if (dlo != dhi) {
        s[MS_LO * n_cells + i] = 0;
        s[MS_HI * n_cells + i] = ~0ull;
        s[MS_MODE * n_cells + i] = MM_EXTREME;
      }
    }
  }
}

// The median outputs (blockIdx.y: the median; output column out0 + blockIdx.y), in the operand's type, valid iff n >= 1:
// the key at rank n / 2 for odd n, else lo.add_wrapping(hi).div_wrapping(2) of the keys at ranks n / 2 - 1 and n / 2.
// f64 NaN results are those of x86-64 SSE arithmetic, on which DataFusion runs: a NaN operand's bits, quieted, the
// first one first; -inf + inf gives the negative default NaN.
__global__ void k_finalize_medians(const uint64_t *state, const MedianCol *meds, const MedianArgs A, uint32_t out0, uint64_t n_cells,
                                   uint64_t bitmap_stride, uint64_t *values, uint8_t *validity) {
  const MedianCol mc = meds[blockIdx.y];
  const uint64_t cell = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  bool valid = false;
  if (cell < n_cells) {
    const uint64_t n = state[mc.count_off + cell];
    const uint64_t *s = A.state + mc.off + cell;
    const uint64_t lo = okey_inv((int64_t)(s[MS_LO * n_cells] ^ 0x8000000000000000ull), mc.phys_type);
    const uint64_t hi = okey_inv((int64_t)(s[MS_HI * n_cells] ^ 0x8000000000000000ull), mc.phys_type);
    uint64_t v = 0;
    valid = n > 0;
    if (n & 1) {
      v = lo;
    } else if (n) {
      if (mc.phys_type == TSKV_PT_I64) {
        v = (uint64_t)((int64_t)(lo + hi) / 2);
      } else if (mc.phys_type == TSKV_PT_U64) {
        v = (lo + hi) / 2;
      } else {
        const double x = __longlong_as_double((long long)lo), y = __longlong_as_double((long long)hi);
        const double sum = x + y;
        if (isnan(x)) v = lo | 0x0008000000000000ull;
        else if (isnan(y)) v = hi | 0x0008000000000000ull;
        else if (isnan(sum)) v = 0xfff8000000000000ull;
        else v = (uint64_t)__double_as_longlong(sum / 2.0);
      }
    }
    values[(uint64_t)(out0 + blockIdx.y) * n_cells + cell] = v;
  }
  const uint32_t bits = __ballot_sync(FULL, valid);
  if ((threadIdx.x & 31) == 0 && (cell >> 3) < bitmap_stride)
    *reinterpret_cast<uint32_t *>(validity + (uint64_t)(out0 + blockIdx.y) * bitmap_stride + (cell >> 3)) = bits;
}

// ---- counter increases (TSKV_QUERY_N_INCREASES): increase(time, x) over each cell's rows in time order --------------
// A cell holds rows of one series (prepare refuses the rest), and along a series the cells are monotone in time. Pass 1
// (the fused scan) gives every cell's n. k_scan_increase pairs the consecutive selected rows of each page (a lane per
// work item), adds its pairs to the cells' sums and leaves one record: its first and last selected point;
// k_merge_increase leaves one record per merged row of the overlap merge groups. The records of a series do not overlap
// in time: sorted by (increase, slot, first time), k_increase_stitch adds the pair across each boundary whose two points
// share a cell. The sums are sections of the exchange region's integer / f64 sum sections.
struct IncreaseCol {
  uint64_t count_off;  // the operand's COUNT section (validity)
  uint64_t off;        // the increase's sum section
  uint32_t qcol;       // the operand's column in the scan's column table (its work-list buckets, its merged values)
  uint16_t column_id;
  uint8_t phys_type;
  uint8_t pad;
};
// The records of every increase: [n_increases][n_rec] (the operand's work items, bucket by bucket from rec0, then the
// merge rows). A record's sort keys are (increase << slot_bits | slot), ~0 when it holds no point, and its first
// point's time - t_base, clamped to t_mask (the page set's time span: the time sort reads only its bits).
struct IncreaseArgs {
  ulonglong4 *rec;        // first cell, last cell, first value, last value
  uint64_t *slot_key;
  uint64_t *time_key;
  const uint32_t *rec0;   // [n_increases][N_BINS * WL_SUB]: the record of the first item of each of the operand's buckets
  int64_t t_base;
  uint64_t t_mask;
  uint32_t n_rec, slot_bits;
};

// The contribution of value v after prev: v > prev adds v - prev, v < prev adds v (a reset), equal adds nothing, in the
// type's order (f64: totalOrder); integers wrap
__device__ __forceinline__ uint64_t increase_step(uint64_t prev, uint64_t v, uint8_t pt) {
  const int64_t kp = okey(prev, pt), kv = okey(v, pt);
  if (kv == kp) return 0;  // (+0.0 for f64)
  if (pt != TSKV_PT_F64) return kv > kp ? v - prev : v;
  const double x = __longlong_as_double((long long)v), y = __longlong_as_double((long long)prev);
  return (uint64_t)__double_as_longlong(kv > kp ? x - y : x);
}
__device__ __forceinline__ void increase_flush(uint64_t *state, const IncreaseCol &ic, uint64_t cell, uint64_t acc) {
  if (ic.phys_type == TSKV_PT_F64) atomicAdd(reinterpret_cast<double *>(state + ic.off + cell), __longlong_as_double((long long)acc));
  else atomicAdd(reinterpret_cast<unsigned long long *>(state + ic.off + cell), (unsigned long long)acc);
}

// One lane's walk over selected points in time order: the run of pairs in the current cell, and the record's points.
struct IncreaseRun {
  uint64_t first_cell, first_v, cell, v, acc;
  int64_t first_t;
  bool have, pairs;
};
__device__ __forceinline__ void increase_begin(IncreaseRun &r) {
  r.have = r.pairs = false;
  r.first_cell = r.first_v = r.cell = r.v = r.acc = 0;
  r.first_t = 0;
}
__device__ __forceinline__ void increase_add(uint64_t *state, const IncreaseCol &ic, IncreaseRun &r, uint64_t cell, int64_t t, uint64_t v) {
  if (!r.have) {
    r.first_cell = cell;
    r.first_v = v;
    r.first_t = t;
    r.have = true;
  } else if (cell == r.cell) {
    const uint64_t d = increase_step(r.v, v, ic.phys_type);
    r.acc = ic.phys_type == TSKV_PT_F64 ? (uint64_t)__double_as_longlong(__longlong_as_double((long long)r.acc) + __longlong_as_double((long long)d))
                                        : r.acc + d;
    r.pairs = true;
  } else {
    if (r.pairs) increase_flush(state, ic, r.cell, r.acc);
    r.acc = 0;
    r.pairs = false;
  }
  r.cell = cell;
  r.v = v;
}
// Flushes the last run and writes record `k` of increase `inc` (slot: the points' series slot).
__device__ __forceinline__ void increase_end(uint64_t *state, const IncreaseCol &ic, const IncreaseArgs &A, uint32_t inc, uint64_t k,
                                             uint32_t slot, const IncreaseRun &r) {
  if (r.pairs) increase_flush(state, ic, r.cell, r.acc);
  const uint64_t i = (uint64_t)inc * A.n_rec + k;
  if (!r.have) return;  // (the slot keys start at ~0)
  A.rec[i] = make_ulonglong4(r.first_cell, r.cell, r.first_v, r.v);
  A.slot_key[i] = ((uint64_t)inc << A.slot_bits) | slot;
  const uint64_t dt = (uint64_t)r.first_t - (uint64_t)A.t_base;
  A.time_key[i] = r.first_t < A.t_base ? 0 : min(dt, A.t_mask);
}

// One page of an increase's operand (work item `item` of its buckets), decoded with its group's time page row by row and
// selected as the medians select (select_row). Decode errors are pass 1's to report: the lane stops at the first.
template <bool EDGES>
__device__ __forceinline__ void increase_page(const ScanParams &P, const IncreaseCol &ic, const IncreaseArgs &A, uint32_t inc,
                                              uint32_t item, uint32_t rec) {
  const uint32_t page = P.work_page[item], slot = P.work_slot[item];
  const tskv_page_desc vd = P.descs[page];
  const uint32_t tpage = P.time_page_of[page];
  const tskv_page_desc td = P.descs[tpage];
  IncreaseRun run;
  increase_begin(run);
  if (vd.phys_type != ic.phys_type || kind_status(vd.reserved) != TSKV_OK || kind_status(td.reserved) != TSKV_OK ||
      td.reserved == DK_ALLNULL || vd.reserved == DK_ALLNULL)
    return;
  PageView tpv, vpv;
  tpv.open(P.arena, td);
  vpv.open(P.arena, vd);
  BitCursor tb, vb;
  tb.init(tpv.bitset);
  vb.init(vpv.bitset);
  DeltaCursor<-1> tc;
  AnyCursor<> vc;
  if (tc.open(tpv, td.reserved) != TSKV_OK || vc.open(vpv, vd.reserved) != TSKV_OK) return;
  const uint4 none = make_uint4(0, 0, 0, 0);
  const uint4 tv4 = P.has_tomb ? tomb_lookup(P, vd.series_id, ic.column_id) : none;
  const uint32_t *keepw = P.row_keep ? P.row_keep + P.keep_off[tpage] : nullptr;
  const uint64_t group_base = group_cell_base<EDGES>(P, slot);
  BucketState bk; bk.valid = false; bk.floor_regime = false; bk.lo = 0; bk.hi = 0; bk.idx = 0;
  int64_t t = 0;
  const uint32_t n_rows = vd.num_values;
  for (uint32_t r = 0; r < n_rows; r++) {
    const bool tv = tb.next(r), vv = vb.next(r);
    uint64_t v = 0;
    if (tv) { t = (int64_t)tc.next(); if (tc.exhausted) break; }
    else if (r == 0) tc.skip_first_if_s8b_sc();
    if (vv) { v = vc.next(); if (vc.failed()) break; }
    else if (r == 0 && !vc.is_gorilla) vc.d.skip_first_if_s8b_sc();
    uint64_t cell;
    if (!(tv && vv) || !select_row<EDGES>(P, keepw, r, t, tv4, none, group_base, bk, cell)) continue;
    increase_add(P.state, ic, run, cell, t, v);
  }
  increase_end(P.state, ic, A, inc, rec, slot, run);
}

// The pages of the increases (blockIdx.y: the increase): one lane per work item of the operand's buckets (every bin,
// wide and narrow), the items pass 1 read; item i of a bucket is record rec0 + i.
template <bool EDGES>
__global__ void __launch_bounds__(128) k_scan_increase(const __grid_constant__ ScanParams P, const IncreaseCol *incs, const IncreaseArgs A) {
  const IncreaseCol ic = incs[blockIdx.y];
  const uint32_t stride = gridDim.x * blockDim.x, t0 = blockIdx.x * blockDim.x + threadIdx.x;
  for (uint32_t b = 0; b < N_BINS; b++)
    for (uint32_t sub = 0; sub < WL_SUB; sub++) {
      const uint32_t k = (b * P.n_cols + ic.qcol) * WL_SUB + sub;
      const uint32_t start = __ldg(P.region_start + k), fill = __ldg(P.region_fill + k);
      const uint32_t r0 = __ldg(A.rec0 + (blockIdx.y * N_BINS + b) * WL_SUB + sub);
      for (uint32_t i = t0; i < fill; i += stride) increase_page<EDGES>(P, ic, A, blockIdx.y, start + i, r0 + i);
    }
}

// Before the record kernels: every record empty, and the identity permutation the sorts start from.
__global__ void k_increase_init(const IncreaseArgs A, uint64_t n, uint32_t *idx) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    A.slot_key[i] = ~0ull;
    A.time_key[i] = 0;
    idx[i] = (uint32_t)i;
  }
}

// Between the two sorts: the slot keys in time order (out[j] = key[idx[j]]).
__global__ void k_increase_gather(const uint64_t *key, const uint32_t *idx, uint64_t n, uint64_t *out) {
  for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (uint64_t)gridDim.x * blockDim.x) out[j] = key[idx[j]];
}

// After the sorts (records in (increase, slot, first time) order, empty ones last): each record whose predecessor holds
// the same increase and slot, and whose first point lies in the predecessor's last cell, adds that pair to the cell.
__global__ void k_increase_stitch(uint64_t *state, const IncreaseCol *incs, const IncreaseArgs A, const uint64_t *slot_sorted,
                                  const uint32_t *idx, uint64_t n) {
  for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x + 1; j < n; j += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t key = slot_sorted[j];
    if (key == ~0ull || slot_sorted[j - 1] != key) continue;
    const ulonglong4 a = A.rec[idx[j - 1]], b = A.rec[idx[j]];
    if (a.y != b.x) continue;
    const IncreaseCol ic = incs[key >> A.slot_bits];
    increase_flush(state, ic, b.x, increase_step(a.w, b.z, ic.phys_type));
  }
}

// The increase outputs (blockIdx.y: the increase; output column out0 + blockIdx.y), in the operand's type, valid iff the
// cell holds a value of the operand.
__global__ void k_finalize_increases(const uint64_t *state, const IncreaseCol *incs, uint32_t out0, uint64_t n_cells, uint64_t bitmap_stride,
                                     uint64_t *values, uint8_t *validity) {
  const IncreaseCol ic = incs[blockIdx.y];
  const uint64_t cell = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  bool valid = false;
  if (cell < n_cells) {
    valid = state[ic.count_off + cell] > 0;
    values[(uint64_t)(out0 + blockIdx.y) * n_cells + cell] = valid ? state[ic.off + cell] : 0;
  }
  const uint32_t bits = __ballot_sync(FULL, valid);
  if ((threadIdx.x & 31) == 0 && (cell >> 3) < bitmap_stride)
    *reinterpret_cast<uint32_t *>(validity + (uint64_t)(out0 + blockIdx.y) * bitmap_stride + (cell >> 3)) = bits;
}

// ---- modes and distinct counts (TSKV_QUERY_N_MODES / _N_DISTINCTS): every cell's selected order keys, sorted ---------
// One gather per distinct operand column id. Pass 1 (the fused scan) gives every cell's n; an exclusive sum of the n over
// the (gather, cell) segments gives segment s the slice [off[s], off[s + 1]) of one key buffer (off[n_segs]: the keys of
// all). k_scan_mode (a lane per page) and k_merge_mode_rows (a thread per merge row) write each selected value's order
// key (median_ukey: one to one on bit patterns, so equal keys are equal values) and its segment into the slice through
// the segment's cursor. Two radix sorts order the buffer by (segment, key); the slots past off[n_segs] hold segment ~0
// and sort last. A run is a stretch of equal (segment, key): k_mode_heads marks each run's first position, a max-scan
// carries it to the run's every position, and k_mode_runs counts each segment's runs (its distinct values) and keeps its
// longest run, of tied lengths the first (the smallest key).
struct ModeGather {
  uint64_t count_off;  // the operand's COUNT section (its pass-1 n)
  uint32_t qcol;       // the operand's column in the scan's column table (its work-list buckets, its merged values)
  uint16_t column_id;
  uint8_t phys_type;
  uint8_t pad;
};
// One mode or distinct output: its gather, and whether it is a distinct count (else a mode).
struct ModeOut {
  uint32_t gather;
  uint32_t distinct;
};
struct ModeArgs {
  uint64_t *keys;            // [bound] the slices k_scan_mode fills; after the sorts, the sorted keys
  uint32_t *segs;            // [bound] their segments (~0: no key); after the sorts, the sorted segments
  int32_t *off;              // [n_segs + 1]
  int32_t *cursor;           // [n_segs] the next free slot of each slice
  unsigned long long *best;  // [n_segs] the longest run: length << 32 | ~(its first position)
  unsigned long long *runs;  // [n_segs] the number of runs
  int32_t *status;           // the scan's status slot and error page
  unsigned long long *err_page;
  uint64_t n_cells, n_segs, bound;
};
struct ModeMax {  // the run starts' max-scan
  __device__ __forceinline__ uint32_t operator()(uint32_t a, uint32_t b) const { return a > b ? a : b; }
};
constexpr uint32_t MODE_STAGE = 16;  // keys a lane stages per slot reservation
constexpr uint32_t MODE_ITEMS = 16;  // sorted positions per lane in k_mode_runs

// A slice that receives more keys than its pass-1 n, or ends with fewer (only a decode error pass 1 reports first can
// cause either): TSKV_ERR_BITSET_MISMATCH, page ~0.
__device__ __forceinline__ void mode_mismatch(const ModeArgs &A) {
  if (atomicCAS(A.status, 0, (int)TSKV_ERR_BITSET_MISMATCH) == 0) *A.err_page = ~0ull;
}
// Reserves n slots of segment seg's slice; false (and the error) when they do not fit it.
__device__ __forceinline__ bool mode_reserve(const ModeArgs &A, uint64_t seg, uint32_t n, uint32_t &pos) {
  pos = (uint32_t)atomicAdd(A.cursor + seg, (int)n);
  const uint32_t end = (uint32_t)A.off[seg + 1];
  if (pos + (uint64_t)n > end || end > A.bound) {
    mode_mismatch(A);
    return false;
  }
  return true;
}

// One lane's staged keys of one segment (stage: the CTA's [MODE_STAGE][128] buffer, column threadIdx.x).
struct ModeRun {
  uint64_t seg;
  uint32_t n;
};
__device__ __forceinline__ void mode_flush(const ModeArgs &A, uint64_t (*stage)[128], ModeRun &r) {
  uint32_t pos;
  if (r.n && mode_reserve(A, r.seg, r.n, pos))
    for (uint32_t k = 0; k < r.n; k++) {
      A.keys[pos + k] = stage[k][threadIdx.x];
      A.segs[pos + k] = (uint32_t)r.seg;
    }
  r.n = 0;
}

// One page of a gather's operand (work item `item` of its buckets), decoded with its group's time page row by row and
// selected as the medians select (select_row). Decode errors are pass 1's to report: the lane stops at the first.
template <bool EDGES>
__device__ __forceinline__ void mode_page(const ScanParams &P, const ModeGather &mg, const ModeArgs &A, uint64_t seg0,
                                          uint64_t (*stage)[128], uint32_t item) {
  const uint32_t page = P.work_page[item], slot = P.work_slot[item];
  const tskv_page_desc vd = P.descs[page];
  const uint32_t tpage = P.time_page_of[page];
  const tskv_page_desc td = P.descs[tpage];
  if (vd.phys_type != mg.phys_type || kind_status(vd.reserved) != TSKV_OK || kind_status(td.reserved) != TSKV_OK ||
      td.reserved == DK_ALLNULL || vd.reserved == DK_ALLNULL)
    return;
  PageView tpv, vpv;
  tpv.open(P.arena, td);
  vpv.open(P.arena, vd);
  BitCursor tb, vb;
  tb.init(tpv.bitset);
  vb.init(vpv.bitset);
  DeltaCursor<-1> tc;
  AnyCursor<> vc;
  if (tc.open(tpv, td.reserved) != TSKV_OK || vc.open(vpv, vd.reserved) != TSKV_OK) return;
  const uint4 none = make_uint4(0, 0, 0, 0);
  const uint4 tv4 = P.has_tomb ? tomb_lookup(P, vd.series_id, mg.column_id) : none;
  const uint32_t *keepw = P.row_keep ? P.row_keep + P.keep_off[tpage] : nullptr;
  const uint64_t group_base = group_cell_base<EDGES>(P, slot);
  BucketState bk; bk.valid = false; bk.floor_regime = false; bk.lo = 0; bk.hi = 0; bk.idx = 0;
  ModeRun run;
  run.seg = ~0ull;
  run.n = 0;
  int64_t t = 0;
  const uint32_t n_rows = vd.num_values;
  for (uint32_t r = 0; r < n_rows; r++) {
    const bool tv = tb.next(r), vv = vb.next(r);
    uint64_t v = 0;
    if (tv) { t = (int64_t)tc.next(); if (tc.exhausted) break; }
    else if (r == 0) tc.skip_first_if_s8b_sc();
    if (vv) { v = vc.next(); if (vc.failed()) break; }
    else if (r == 0 && !vc.is_gorilla) vc.d.skip_first_if_s8b_sc();
    uint64_t cell;
    if (!(tv && vv) || !select_row<EDGES>(P, keepw, r, t, tv4, none, group_base, bk, cell)) continue;
    if (seg0 + cell != run.seg || run.n == MODE_STAGE) {
      mode_flush(A, stage, run);
      run.seg = seg0 + cell;
    }
    stage[run.n++][threadIdx.x] = median_ukey(v, mg.phys_type);
  }
  mode_flush(A, stage, run);
}

// The gathers' pages (blockIdx.y: the gather): one lane per work item of the operand's buckets (every bin, wide and
// narrow), the items pass 1 read.
template <bool EDGES>
__global__ void __launch_bounds__(128) k_scan_mode(const __grid_constant__ ScanParams P, const ModeGather *gathers, const ModeArgs A) {
  __shared__ uint64_t stage[MODE_STAGE][128];
  const ModeGather mg = gathers[blockIdx.y];
  const uint64_t seg0 = (uint64_t)blockIdx.y * A.n_cells;
  const uint32_t stride = gridDim.x * blockDim.x, t0 = blockIdx.x * blockDim.x + threadIdx.x;
  for (uint32_t k = mg.qcol * WL_SUB; k < N_BINS * P.n_cols * WL_SUB; k += P.n_cols * WL_SUB)
    for (uint32_t sub = 0; sub < WL_SUB; sub++) {
      const uint32_t start = __ldg(P.region_start + k + sub), fill = __ldg(P.region_fill + k + sub);
      for (uint32_t i = t0; i < fill; i += stride) mode_page<EDGES>(P, mg, A, seg0, stage, start + i);
    }
}

// After pass 1: every segment's n (off, summed in place into the slices' starts next), off[n_segs] = 0, and the run
// results cleared.
__global__ void k_mode_counts(const uint64_t *state, const ModeGather *gathers, const ModeArgs A) {
  for (uint64_t s = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; s <= A.n_segs; s += (uint64_t)gridDim.x * blockDim.x) {
    if (s == A.n_segs) { A.off[s] = 0; continue; }
    const uint64_t n = state[gathers[s / A.n_cells].count_off + s % A.n_cells];
    A.off[s] = (int32_t)min(n, (uint64_t)TSKV_MAX_SORTED_ROWS);
    A.best[s] = A.runs[s] = 0;
  }
}

// After the sorts: start[i] = i at the first position of a run, else 0 (a max-scan then gives every position its run's
// first); and every slice whose cursor did not end at its end is an error.
__global__ void k_mode_heads(const ModeArgs A, uint32_t *start) {
  const uint64_t total = min((uint64_t)(uint32_t)A.off[A.n_segs], A.bound), stride = (uint64_t)gridDim.x * blockDim.x;
  const uint64_t t0 = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  for (uint64_t i = t0; i < A.bound; i += stride)
    start[i] = i < total && (i == 0 || A.segs[i] != A.segs[i - 1] || A.keys[i] != A.keys[i - 1]) ? (uint32_t)i : 0;
  for (uint64_t s = t0; s < A.n_segs; s += stride)
    if (A.cursor[s] != A.off[s + 1]) mode_mismatch(A);
}

// After the max-scan: a lane per MODE_ITEMS sorted positions adds, at each run's last position, one run and the run's
// (length, first position) to its segment; a warp combines its lanes' last segments before the atomics.
__global__ void __launch_bounds__(256) k_mode_runs(const ModeArgs A, const uint32_t *start) {
  const uint64_t total = min((uint64_t)(uint32_t)A.off[A.n_segs], A.bound);
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t warps = (uint64_t)gridDim.x * (blockDim.x >> 5);
  for (uint64_t base = (((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5) * 32 * MODE_ITEMS; base < total;
       base += warps * 32 * MODE_ITEMS) {
    uint32_t seg = ~0u, runs = 0;
    unsigned long long best = 0;
    const uint64_t i0 = base + (uint64_t)lane * MODE_ITEMS, i1 = min(i0 + MODE_ITEMS, total);
    for (uint64_t i = i0; i < i1; i++) {
      const uint32_t s = A.segs[i];
      if (i + 1 < total && A.segs[i + 1] == s && A.keys[i + 1] == A.keys[i]) continue;  // not a run's last position
      if (s != seg) {
        if (runs) {
          atomicAdd(A.runs + seg, (unsigned long long)runs);
          atomicMax(A.best + seg, best);
        }
        seg = s;
        runs = 0;
        best = 0;
      }
      const uint32_t first = start[i];
      runs++;
      best = max(best, ((unsigned long long)(i - first + 1) << 32) | (uint32_t)~first);
    }
    const uint32_t group = __match_any_sync(FULL, seg);
    const uint32_t hi = __reduce_max_sync(group, (uint32_t)(best >> 32));
    const uint32_t lo = __reduce_max_sync(group, (uint32_t)(best >> 32) == hi ? (uint32_t)best : 0u);
    const uint32_t n = __reduce_add_sync(group, runs);
    if (seg != ~0u && n && lane == (uint32_t)(__ffs(group) - 1)) {
      atomicAdd(A.runs + seg, (unsigned long long)n);
      atomicMax(A.best + seg, ((unsigned long long)hi << 32) | lo);
    }
  }
}

// The mode and distinct outputs (blockIdx.y: the output; output column out0 + blockIdx.y). A mode is in the operand's
// type, valid iff its cell holds a value: the key of the cell's longest run. A distinct is the cell's number of runs, a
// u64, always valid.
__global__ void k_finalize_modes(const ModeArgs A, const ModeGather *gathers, const ModeOut *outs, uint32_t out0, uint64_t bitmap_stride,
                                 uint64_t *values, uint8_t *validity) {
  const ModeOut mo = outs[blockIdx.y];
  const uint64_t cell = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  bool valid = false;
  if (cell < A.n_cells) {
    const uint64_t s = (uint64_t)mo.gather * A.n_cells + cell;
    uint64_t v = 0;
    if (mo.distinct) {
      v = A.runs[s];
      valid = true;
    } else {
      const uint32_t first = ~(uint32_t)A.best[s];
      valid = A.off[s + 1] > A.off[s] && first < A.bound;
      if (valid) v = okey_inv((int64_t)(A.keys[first] ^ 0x8000000000000000ull), gathers[mo.gather].phys_type);
    }
    values[(uint64_t)(out0 + blockIdx.y) * A.n_cells + cell] = v;
  }
  const uint32_t bits = __ballot_sync(FULL, valid);
  if ((threadIdx.x & 31) == 0 && (cell >> 3) < bitmap_stride)
    *reinterpret_cast<uint32_t *>(validity + (uint64_t)(out0 + blockIdx.y) * bitmap_stride + (cell >> 3)) = bits;
}

// ---- gauges (TSKV_QUERY_N_GAUGES): gauge_agg(time, x), each cell's first two and last two points ----------------------
// Pass 1 (the fused scan) gives every cell's n. k_gauge_scan (a lane per work item of the operand's buckets) and
// k_gauge_merge_rows (a thread per merged row) append one record per (page, cell) run: the run's points as a GaugeAcc.
// A radix sort orders the records by key (gauge, kernel cell), a reduce by key joins each key's records with gauge_join,
// and k_gauge_scatter writes the states of the kernel's grid. A sliding scan's panes fold into windows (k_gauge_fold),
// and the ranks' states join in k_merge_gauges. The order of points is (t, slot): ties of time across series go to the
// lower slot. gauge_join is associative and commutative on disjoint point sets, so the result does not depend on the
// order the records were appended in.
struct GaugeCol {
  uint64_t count_off;  // the operand's COUNT section (n)
  uint32_t qcol;       // the operand's column in the scan's column table (its work-list buckets, its merged values)
  uint16_t column_id;
  uint8_t phys_type;
  uint8_t pad;
};
// A set of points: cnt = min(points, 2); p[0], p[1] its two smallest under (t, slot), p[2], p[3] its two largest. One
// point fills all four places, two points give p0, p1, p0, p1 (the reference's second is then the last point and its
// penultimate the first). v holds the operand's bit pattern.
struct GaugeAcc {
  int64_t t[4];
  uint64_t v[4];
  uint32_t s[4];
  uint64_t cnt;
};
static_assert(sizeof(GaugeAcc) == 88, "a gauge state is 11 words of the exchange region");
constexpr uint32_t GAUGE_WORDS = sizeof(GaugeAcc) / 8;
constexpr uint32_t GAUGE_OUTS = 9;  // n, then (t, v) of first, second, penultimate, last

__host__ __device__ __forceinline__ bool gauge_before(const GaugeAcc &a, int i, const GaugeAcc &b, int j) {
  return a.t[i] < b.t[j] || (a.t[i] == b.t[j] && a.s[i] < b.s[j]);
}
__host__ __device__ __forceinline__ void gauge_put(GaugeAcc &r, int i, const GaugeAcc &a, int j) {
  r.t[i] = a.t[j];
  r.v[i] = a.v[j];
  r.s[i] = a.s[j];
}
// The points of a and b (disjoint sets). The smallest is the smaller of the two first points; the second smallest the
// smaller of the other first point and the winner's second (the loser's second is past its own first). The same for the
// two largest.
__host__ __device__ __forceinline__ GaugeAcc gauge_join(const GaugeAcc &a, const GaugeAcc &b) {
  if (!b.cnt) return a;
  if (!a.cnt) return b;
  GaugeAcc r;
  r.cnt = 2;
  if (gauge_before(a, 0, b, 0)) {
    gauge_put(r, 0, a, 0);
    if (a.cnt >= 2 && gauge_before(a, 1, b, 0)) gauge_put(r, 1, a, 1);
    else gauge_put(r, 1, b, 0);
  } else {
    gauge_put(r, 0, b, 0);
    if (b.cnt >= 2 && gauge_before(b, 1, a, 0)) gauge_put(r, 1, b, 1);
    else gauge_put(r, 1, a, 0);
  }
  if (gauge_before(b, 3, a, 3)) {
    gauge_put(r, 3, a, 3);
    if (a.cnt >= 2 && gauge_before(b, 3, a, 2)) gauge_put(r, 2, a, 2);
    else gauge_put(r, 2, b, 3);
  } else {
    gauge_put(r, 3, b, 3);
    if (b.cnt >= 2 && gauge_before(a, 3, b, 2)) gauge_put(r, 2, b, 2);
    else gauge_put(r, 2, a, 3);
  }
  return r;
}
struct GaugeJoin {
  __host__ __device__ __forceinline__ GaugeAcc operator()(const GaugeAcc &a, const GaugeAcc &b) const { return gauge_join(a, b); }
};
__device__ __forceinline__ GaugeAcc gauge_point(int64_t t, uint32_t slot, uint64_t v) {
  GaugeAcc r;
  for (int i = 0; i < 4; i++) {
    r.t[i] = t;
    r.v[i] = v;
    r.s[i] = slot;
  }
  r.cnt = 1;
  return r;
}

// The records and the buffers of the sort and the reduce, all sized at prepare (bound records).
struct GaugeArgs {
  GaugeAcc *rec;        // [bound] appended records
  GaugeAcc *sorted;     // [bound] the records in key order (empty past the last key)
  GaugeAcc *agg;        // [bound] the reduce's joined states, one per key
  uint64_t *key;        // [2 * bound] the records' keys (~0: no record), then the sorted keys
  uint32_t *idx;        // [2 * bound] the records' positions, then in key order
  uint64_t *uniq;       // [bound] the reduce's keys
  int32_t *n_runs;      // the reduce's number of keys
  unsigned int *n_rec;  // the append counter
  GaugeAcc *dst;        // [n_segs] the states of the kernels' grid (a sliding scan: its panes)
  int32_t *status;      // the scan's status slot and error page
  unsigned long long *err_page;
  uint64_t kern_cells, n_segs, bound;
};

// A cell whose records disagree with its pass-1 n, or records past the bound (only a decode error pass 1 reports first
// can cause either): TSKV_ERR_BITSET_MISMATCH, page ~0.
__device__ __forceinline__ void gauge_mismatch(int32_t *status, unsigned long long *err_page) {
  if (atomicCAS(status, 0, (int)TSKV_ERR_BITSET_MISMATCH) == 0) *err_page = ~0ull;
}
// Appends record r of key `key`: the converged lanes of the warp take their places with one atomic.
__device__ __forceinline__ void gauge_emit(const GaugeArgs &A, uint64_t key, const GaugeAcc &r) {
  const uint32_t m = __activemask(), lane = threadIdx.x & 31, leader = __ffs(m) - 1;
  const uint32_t rank = __popc(m & ((1u << lane) - 1));
  uint32_t base = 0;
  if (lane == leader) base = atomicAdd(A.n_rec, (unsigned int)__popc(m));
  const uint32_t pos = __shfl_sync(m, base, leader) + rank;
  if (pos >= A.bound) {
    gauge_mismatch(A.status, A.err_page);
    return;
  }
  A.key[pos] = key;
  A.idx[pos] = pos;
  A.rec[pos] = r;
}

// One page of a gauge's operand (work item `item` of its buckets), decoded with its group's time page row by row and
// selected as the medians select (select_row): one record per run of selected rows in one cell. Decode errors are pass
// 1's to report: the lane stops at the first.
template <bool EDGES>
__device__ __forceinline__ void gauge_page(const ScanParams &P, const GaugeCol &gc, const GaugeArgs &A, uint64_t key0, uint32_t item) {
  const uint32_t page = P.work_page[item], slot = P.work_slot[item];
  const tskv_page_desc vd = P.descs[page];
  const uint32_t tpage = P.time_page_of[page];
  const tskv_page_desc td = P.descs[tpage];
  if (vd.phys_type != gc.phys_type || kind_status(vd.reserved) != TSKV_OK || kind_status(td.reserved) != TSKV_OK ||
      td.reserved == DK_ALLNULL || vd.reserved == DK_ALLNULL)
    return;
  PageView tpv, vpv;
  tpv.open(P.arena, td);
  vpv.open(P.arena, vd);
  BitCursor tb, vb;
  tb.init(tpv.bitset);
  vb.init(vpv.bitset);
  DeltaCursor<-1> tc;
  AnyCursor<> vc;
  if (tc.open(tpv, td.reserved) != TSKV_OK || vc.open(vpv, vd.reserved) != TSKV_OK) return;
  const uint4 none = make_uint4(0, 0, 0, 0);
  const uint4 tv4 = P.has_tomb ? tomb_lookup(P, vd.series_id, gc.column_id) : none;
  const uint32_t *keepw = P.row_keep ? P.row_keep + P.keep_off[tpage] : nullptr;
  const uint64_t group_base = group_cell_base<EDGES>(P, slot);
  BucketState bk; bk.valid = false; bk.floor_regime = false; bk.lo = 0; bk.hi = 0; bk.idx = 0;
  GaugeAcc run;
  run.cnt = 0;
  uint64_t run_cell = 0;
  int64_t t = 0;
  const uint32_t n_rows = vd.num_values;
  for (uint32_t r = 0; r < n_rows; r++) {
    const bool tv = tb.next(r), vv = vb.next(r);
    uint64_t v = 0;
    if (tv) { t = (int64_t)tc.next(); if (tc.exhausted) break; }
    else if (r == 0) tc.skip_first_if_s8b_sc();
    if (vv) { v = vc.next(); if (vc.failed()) break; }
    else if (r == 0 && !vc.is_gorilla) vc.d.skip_first_if_s8b_sc();
    uint64_t cell;
    if (!(tv && vv) || !select_row<EDGES>(P, keepw, r, t, tv4, none, group_base, bk, cell)) continue;
    if (run.cnt && cell != run_cell) {
      gauge_emit(A, key0 + run_cell, run);
      run.cnt = 0;
    }
    run_cell = cell;
    run = gauge_join(run, gauge_point(t, slot, v));
  }
  if (run.cnt) gauge_emit(A, key0 + run_cell, run);
}

// The gauges' pages (blockIdx.y: the gauge): one lane per work item of the operand's buckets (every bin, wide and
// narrow), the items pass 1 read.
template <bool EDGES>
__global__ void __launch_bounds__(128) k_gauge_scan(const __grid_constant__ ScanParams P, const GaugeCol *gcols, const GaugeArgs A) {
  const GaugeCol gc = gcols[blockIdx.y];
  const uint64_t key0 = (uint64_t)blockIdx.y * A.kern_cells;
  const uint32_t stride = gridDim.x * blockDim.x, t0 = blockIdx.x * blockDim.x + threadIdx.x;
  for (uint32_t k = gc.qcol * WL_SUB; k < N_BINS * P.n_cols * WL_SUB; k += P.n_cols * WL_SUB)
    for (uint32_t sub = 0; sub < WL_SUB; sub++) {
      const uint32_t start = __ldg(P.region_start + k + sub), fill = __ldg(P.region_fill + k + sub);
      for (uint32_t i = t0; i < fill; i += stride) gauge_page<EDGES>(P, gc, A, key0, start + i);
    }
}

// After the sort: the records in key order; positions past the last record (key ~0) hold an empty state.
__global__ void k_gauge_gather(const GaugeArgs A) {
  const uint64_t *skey = A.key + A.bound;
  const uint32_t *sidx = A.idx + A.bound;
  for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < A.bound; j += (uint64_t)gridDim.x * blockDim.x) {
    if (skey[j] < A.n_segs) {
      A.sorted[j] = A.rec[sidx[j]];
    } else {
      GaugeAcc e{};
      A.sorted[j] = e;
    }
  }
}

// After the reduce: every key's joined state into the grid's states (cleared before).
__global__ void k_gauge_scatter(const GaugeArgs A) {
  const uint64_t n = (uint64_t)max(*A.n_runs, 0);
  for (uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (uint64_t)gridDim.x * blockDim.x)
    if (A.uniq[r] < A.n_segs) A.dst[A.uniq[r]] = A.agg[r];
}

// Sliding windows: window j of a group joins its panes j - k + 1 .. j (those that exist), as k_window_combine folds.
__global__ void k_gauge_fold(const GaugeAcc *pane, GaugeAcc *win, uint32_t n_gauges, uint32_t n_groups, uint32_t n_windows,
                             uint32_t n_panes, uint32_t k) {
  const uint64_t n = (uint64_t)n_gauges * n_groups * n_windows;
  for (uint64_t c = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; c < n; c += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t g = c / n_windows;  // (gauge, group)
    const uint32_t j = (uint32_t)(c - g * n_windows);
    const uint32_t p0 = j + 1 >= k ? j + 1 - k : 0, p1 = j < n_panes - 1 ? j : n_panes - 1;
    GaugeAcc acc;
    acc.cnt = 0;
    for (uint32_t p = p0; p <= p1; p++) acc = gauge_join(acc, pane[g * n_panes + p]);
    win[c] = acc;
  }
}

// Every cell of every gauge (the query's grid): a state without a pass-1 n, or an n without a state, is an error.
__global__ void k_gauge_check(const uint64_t *state, const GaugeCol *gcols, const GaugeAcc *gs, uint32_t n_gauges, uint64_t n_cells,
                              int32_t *status, unsigned long long *err_page) {
  const uint64_t n = (uint64_t)n_gauges * n_cells;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t g = i / n_cells, cell = i - g * n_cells;
    if ((gs[i].cnt != 0) != (state[gcols[g].count_off + cell] != 0)) gauge_mismatch(status, err_page);
  }
}

// Multi-GPU, after k_merge_gathered: every gauge state joins the ranks' states (the gauge section at off, n states).
__global__ void k_merge_gauges(uint64_t *state, uint64_t off, uint64_t n, const uint64_t *gathered, uint32_t n_ranks, uint64_t exch_words) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    GaugeAcc acc;
    acc.cnt = 0;
    for (uint32_t r = 0; r < n_ranks; r++)
      acc = gauge_join(acc, reinterpret_cast<const GaugeAcc *>(gathered + r * exch_words + off)[i]);
    reinterpret_cast<GaugeAcc *>(state + off)[i] = acc;
  }
}

// The gauge outputs (blockIdx.y: gauge * GAUGE_OUTS + output; output column out0 + blockIdx.y): n (u64, always valid),
// then t (i64) and v (f64: integers rounded to nearest) of the first, second, penultimate and last point, valid iff n >= 1.
__global__ void k_finalize_gauges(const uint64_t *state, const GaugeCol *gcols, uint64_t off, uint32_t out0, uint64_t n_cells,
                                  uint64_t bitmap_stride, uint64_t *values, uint8_t *validity) {
  const uint32_t g = blockIdx.y / GAUGE_OUTS, f = blockIdx.y % GAUGE_OUTS;
  const GaugeCol gc = gcols[g];
  const uint64_t cell = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  bool valid = false;
  if (cell < n_cells) {
    const uint64_t n = state[gc.count_off + cell];
    uint64_t v = n;
    valid = f == 0 || n != 0;
    if (f && valid) {
      const GaugeAcc &a = reinterpret_cast<const GaugeAcc *>(state + off)[(uint64_t)g * n_cells + cell];
      const uint32_t p = (f - 1) >> 1;
      if (((f - 1) & 1) == 0) {
        v = (uint64_t)a.t[p];
      } else {
        v = a.v[p];
        if (gc.phys_type == TSKV_PT_I64) v = (uint64_t)__double_as_longlong(__ll2double_rn((long long)v));
        else if (gc.phys_type == TSKV_PT_U64) v = (uint64_t)__double_as_longlong(__ull2double_rn((unsigned long long)v));
      }
    }
    values[(uint64_t)(out0 + blockIdx.y) * n_cells + cell] = valid ? v : 0;
  }
  const uint32_t bits = __ballot_sync(FULL, valid);
  if ((threadIdx.x & 31) == 0 && (cell >> 3) < bitmap_stride)
    *reinterpret_cast<uint32_t *>(validity + (uint64_t)(out0 + blockIdx.y) * bitmap_stride + (cell >> 3)) = bits;
}

// ---- state aggs (TSKV_QUERY_N_STATE_AGGS): compact_state_agg(time, x), the time each cell spends in every state ----------
// A cell holds rows of one series (prepare refuses the rest), and along a series the cells are monotone in time. Every
// selected row is a point (t, state), a NULL value (the page's bitmap, a column tombstone, a merged row without a value)
// a state of its own. Each pair of consecutive points adds t' - t to the earlier point's state. Pass 1 (the fused scan)
// counts each cell's non-NULL rows. k_state_scan (a lane per work item of the operand's buckets) walks a page's points:
// a run of one state that ends at the next run's first point appends one duration record (segment, state key, t' - t0),
// and at a cell change or at the page's end the open run appends its partial duration (last t - t0) and the (page, cell)
// piece appends a boundary record (its first time, its last time and state). k_state_merge_rows does the same for every
// merged row of the overlap merge groups. Sorted by first time, then stably by (agg, slot), consecutive boundary records
// of one cell add the gap between them to the earlier one's last state (k_state_stitch). Since every piece already gave
// its last state an entry, the reference's finalize (a 0 entry for the cell's final state) needs no record of its own.
// Two radix sorts order the duration records by (segment, state key), a reduce by key sums each key's durations: its
// unique keys are the cells' map entries in output order. A segment is (agg, cell) << 1 | non-NULL, so that the NULL
// state comes first; the state key is the operand's order key (i64: sign bit flipped; u64: itself).
struct StateCol {
  uint64_t count_off;  // the operand's COUNT section (the cell's non-NULL rows)
  uint32_t qcol;       // the operand's column in the scan's column table (its work-list buckets, its merged values)
  uint16_t column_id;
  uint8_t phys_type;
  uint8_t periods;     // the operand's agg_mask is TSKV_STATE_PERIODS: the agg returns its periods too
};
// One map entry's key: the segment and the state key.
struct StateKey {
  uint64_t seg, key;
  __host__ __device__ __forceinline__ bool operator==(const StateKey &o) const { return seg == o.seg && key == o.key; }
};
// One (page, cell) piece of a slot's points: its first time, its last time and its last state.
struct StateBound {
  int64_t first_t, last_t;
  uint64_t seg, key;  // the last state's segment and key
};
// The records and the buffers of the sorts and the reduce, all sized at prepare: dbound duration records, bbound
// boundary records.
struct StateArgs {
  uint64_t *seg;        // [2 * dbound] the duration records' segments (~0: no record; sorted after the sorts), then in key order
  uint64_t *key;        // [2 * dbound] their state keys, then sorted
  int64_t *dur;         // [dbound] their durations
  int64_t *start;       // [dbound] their start times (null: no operand has TSKV_STATE_PERIODS, nothing is written)
  uint32_t *idx;        // [2 * dbound] positions: identity (the (segment, key) order after the sorts), then key order
  StateKey *skey;       // [dbound] the records' keys in (segment, key) order (segment ~0 past the last record)
  int64_t *sdur;        // [dbound] their durations
  StateKey *uniq;       // [dbound] the reduce's keys
  int64_t *sum;         // [dbound] the reduce's sums
  int32_t *n_runs;      // the reduce's number of keys
  unsigned int *n_dur;  // the duration records' append counter
  unsigned int *n_bnd;  // the boundary records' append counter
  StateBound *bnd;      // [bbound] boundary records
  uint64_t *bkey;       // [5 * bbound] slot keys | time keys | time keys sorted | slot keys in time order | slot keys sorted
  uint32_t *bidx;       // [3 * bbound] identity | time order | (agg, slot, first time) order
  uint64_t *rows;       // [n_segs] the non-NULL rows the records saw, per (agg, cell)
  uint32_t *off;        // [n_segs + 1] the entries per (agg, cell), then their exclusive sum (the CSR offsets)
  int32_t *status;      // the scan's status slot and error page
  unsigned long long *err_page;
  uint64_t n_cells, n_segs, dbound, bbound;
  int64_t t_base;       // boundary time keys: first time - t_base, clamped to t_mask (the page set's time span)
  uint64_t t_mask;
  uint32_t slot_bits;   // boundary slot keys: agg << slot_bits | slot
};

struct StateSum {
  __host__ __device__ __forceinline__ int64_t operator()(int64_t a, int64_t b) const { return a + b; }
};

__device__ __forceinline__ uint64_t state_key(uint64_t v, uint8_t pt) { return pt == TSKV_PT_I64 ? v ^ 0x8000000000000000ull : v; }
__device__ __forceinline__ uint64_t state_seg(uint64_t agg_cell, bool null) { return (agg_cell << 1) | (null ? 0u : 1u); }

// Appends a duration record [t, t + d): the converged lanes of the warp take their places with one atomic.
__device__ __forceinline__ void state_emit(const StateArgs &A, uint64_t seg, uint64_t key, int64_t t, int64_t d) {
  const uint32_t m = __activemask(), lane = threadIdx.x & 31, leader = __ffs(m) - 1;
  uint32_t base = 0;
  if (lane == leader) base = atomicAdd(A.n_dur, (unsigned int)__popc(m));
  const uint32_t pos = __shfl_sync(m, base, leader) + __popc(m & ((1u << lane) - 1));
  if (pos >= A.dbound) {
    gauge_mismatch(A.status, A.err_page);
    return;
  }
  A.seg[pos] = seg;
  A.key[pos] = key;
  A.dur[pos] = d;
  if (A.start) A.start[pos] = t;
}
// Appends a boundary record of slot `slot` (agg: the record's state agg) and the piece's non-NULL row count.
__device__ __forceinline__ void state_bound(const StateArgs &A, uint32_t agg, uint32_t slot, const StateBound &b, uint64_t nn) {
  const uint32_t m = __activemask(), lane = threadIdx.x & 31, leader = __ffs(m) - 1;
  uint32_t base = 0;
  if (lane == leader) base = atomicAdd(A.n_bnd, (unsigned int)__popc(m));
  const uint32_t pos = __shfl_sync(m, base, leader) + __popc(m & ((1u << lane) - 1));
  if (nn) atomicAdd(reinterpret_cast<unsigned long long *>(A.rows + (b.seg >> 1)), (unsigned long long)nn);
  if (pos >= A.bbound) {
    gauge_mismatch(A.status, A.err_page);
    return;
  }
  A.bnd[pos] = b;
  A.bkey[pos] = ((uint64_t)agg << A.slot_bits) | slot;
  const uint64_t dt = (uint64_t)b.first_t - (uint64_t)A.t_base;
  A.bkey[A.bbound + pos] = b.first_t < A.t_base ? 0 : min(dt, A.t_mask);
}

// One lane's walk over a piece of points in time order: the open run and the piece.
struct StateRun {
  StateBound b;    // the piece: first time, last time, the open run's state
  int64_t run_t;   // the open run's first time
  uint64_t nn;     // the piece's non-NULL rows
  bool open;
};
__device__ __forceinline__ void state_close(const StateArgs &A, uint32_t agg, uint32_t slot, StateRun &r) {
  if (!r.open) return;
  state_emit(A, r.b.seg, r.b.key, r.run_t, r.b.last_t - r.run_t);
  state_bound(A, agg, slot, r.b, r.nn);
  r.open = false;
}
__device__ __forceinline__ void state_add(const StateArgs &A, uint32_t agg, uint32_t slot, StateRun &r, uint64_t cell, int64_t t,
                                          bool null, uint64_t key) {
  const uint64_t seg = state_seg((uint64_t)agg * A.n_cells + cell, null);
  if (r.open && (r.b.seg >> 1) != (seg >> 1)) state_close(A, agg, slot, r);
  if (!r.open) {
    r.open = true;
    r.b.first_t = t;
    r.nn = 0;
  } else if (r.b.seg != seg || r.b.key != key) {
    state_emit(A, r.b.seg, r.b.key, r.run_t, t - r.run_t);
  } else {
    r.b.last_t = t;
    r.nn += !null;
    return;
  }
  r.b.seg = seg;
  r.b.key = key;
  r.run_t = t;
  r.b.last_t = t;
  r.nn += !null;
}

// One page of a state agg's operand (work item `item` of its buckets), decoded with its group's time page row by row and
// selected as the medians select (select_row) except that the operand's column tombstones make NULL states instead of
// dropping the row. Decode errors are pass 1's to report: the lane stops at the first.
template <bool EDGES>
__device__ __forceinline__ void state_page(const ScanParams &P, const StateCol &sc, const StateArgs &A, uint32_t agg, uint32_t item) {
  const uint32_t page = P.work_page[item], slot = P.work_slot[item];
  const tskv_page_desc vd = P.descs[page];
  const uint32_t tpage = P.time_page_of[page];
  const tskv_page_desc td = P.descs[tpage];
  if (vd.phys_type != sc.phys_type || kind_status(vd.reserved) != TSKV_OK || kind_status(td.reserved) != TSKV_OK ||
      td.reserved == DK_ALLNULL)
    return;
  PageView tpv, vpv;
  tpv.open(P.arena, td);
  vpv.open(P.arena, vd);
  BitCursor tb, vb;
  tb.init(tpv.bitset);
  vb.init(vpv.bitset);
  DeltaCursor<-1> tc;
  AnyCursor<> vc;
  if (tc.open(tpv, td.reserved) != TSKV_OK || vc.open(vpv, vd.reserved) != TSKV_OK) return;
  const bool allnull = vd.reserved == DK_ALLNULL;
  const uint4 none = make_uint4(0, 0, 0, 0);
  const uint4 tv4 = P.has_tomb ? tomb_lookup(P, vd.series_id, sc.column_id) : none;
  const uint4 rows4 = make_uint4(tv4.x, tv4.y, 0, 0);  // (row drops select; the column's ranges make NULL states)
  const uint32_t *keepw = P.row_keep ? P.row_keep + P.keep_off[tpage] : nullptr;
  const uint64_t group_base = group_cell_base<EDGES>(P, slot);
  BucketState bk; bk.valid = false; bk.floor_regime = false; bk.lo = 0; bk.hi = 0; bk.idx = 0;
  StateRun run;
  run.open = false;
  run.b.first_t = run.b.last_t = run.run_t = 0;
  run.b.seg = run.b.key = run.nn = 0;
  int64_t t = 0;
  const uint32_t n_rows = vd.num_values;
  for (uint32_t r = 0; r < n_rows; r++) {
    const bool tv = tb.next(r), vv = vb.next(r) && !allnull;
    uint64_t v = 0;
    if (tv) { t = (int64_t)tc.next(); if (tc.exhausted) break; }
    else if (r == 0) tc.skip_first_if_s8b_sc();
    if (vv) { v = vc.next(); if (vc.failed()) break; }
    else if (r == 0 && !vc.is_gorilla) vc.d.skip_first_if_s8b_sc();
    uint64_t cell;
    if (!tv || !select_row<EDGES>(P, keepw, r, t, rows4, none, group_base, bk, cell)) continue;
    bool null = !vv;
    if (!null && tv4.w) {
      int64_t lo = INT64_MIN, hi = INT64_MAX;
      null = tomb_span(P.tomb_ranges + tv4.z, tv4.w, t, lo, hi);
    }
    state_add(A, agg, slot, run, cell, t, null, null ? 0 : state_key(v, sc.phys_type));
  }
  state_close(A, agg, slot, run);
}

// The state aggs' pages (blockIdx.y: the state agg): one lane per work item of the operand's buckets (every bin, wide and
// narrow), the items pass 1 read. (A minimum of one block per SM lets ptxas keep the walk in registers: with the
// default it settles on 128 registers and spills.)
template <bool EDGES>
__global__ void __launch_bounds__(128, 1) k_state_scan(const __grid_constant__ ScanParams P, const StateCol *scols, const StateArgs A) {
  const StateCol sc = scols[blockIdx.y];
  const uint32_t stride = gridDim.x * blockDim.x, t0 = blockIdx.x * blockDim.x + threadIdx.x;
  for (uint32_t k = sc.qcol * WL_SUB; k < N_BINS * P.n_cols * WL_SUB; k += P.n_cols * WL_SUB)
    for (uint32_t sub = 0; sub < WL_SUB; sub++) {
      const uint32_t start = __ldg(P.region_start + k + sub), fill = __ldg(P.region_fill + k + sub);
      for (uint32_t i = t0; i < fill; i += stride) state_page<EDGES>(P, sc, A, blockIdx.y, start + i);
    }
}

// Before the record kernels: no boundary record, the identity permutations the sorts start from.
__global__ void k_state_init(const StateArgs A) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < A.bbound; i += (uint64_t)gridDim.x * blockDim.x) {
    A.bkey[i] = ~0ull;
    A.bkey[A.bbound + i] = 0;
    A.bidx[i] = (uint32_t)i;
  }
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < A.dbound; i += (uint64_t)gridDim.x * blockDim.x) {
    A.seg[i] = ~0ull;
    A.key[i] = ~0ull;
    A.dur[i] = 0;
    A.idx[i] = (uint32_t)i;
  }
}

// After the boundary sorts (records in (agg, slot, first time) order, empty ones last): a record whose successor holds
// the same agg and slot and starts in the same cell adds the gap to its last state.
__global__ void k_state_stitch(const StateArgs A) {
  const uint64_t *slot_sorted = A.bkey + 4 * A.bbound;
  const uint32_t *order = A.bidx + 2 * A.bbound;
  for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x + 1; j < A.bbound; j += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t key = slot_sorted[j];
    if (key == ~0ull || slot_sorted[j - 1] != key) continue;
    const StateBound a = A.bnd[order[j - 1]], b = A.bnd[order[j]];
    if ((a.seg >> 1) != (b.seg >> 1)) continue;
    state_emit(A, a.seg, a.key, a.last_t, b.first_t - a.last_t);
  }
}

// Between the two sorts of the boundary records (out[j] = key[idx[j]]) and of the duration records (the segments in key
// order): one gather.
__global__ void k_state_gather(const uint64_t *key, const uint32_t *idx, uint64_t n, uint64_t *out) {
  for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (uint64_t)gridDim.x * blockDim.x) out[j] = key[idx[j]];
}

// After the duration sorts (the sorted segments and the final order over the records' own): the records' (segment, key)
// and durations in that order.
__global__ void k_state_order(const StateArgs A) {
  for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < A.dbound; j += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t i = A.idx[j];
    StateKey k;
    k.seg = A.seg[j];
    k.key = A.key[i];
    A.skey[j] = k;
    A.sdur[j] = A.dur[i];
  }
}

// After the reduce: each (agg, cell)'s entries (the unique keys past the last cell's, segment ~0, are not entries).
__global__ void k_state_count(const StateArgs A) {
  const uint64_t n = (uint64_t)max(*A.n_runs, 0);
  for (uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t s = A.uniq[r].seg >> 1;
    if (s < A.n_segs) atomicAdd(A.off + s, 1u);
  }
}

// Every cell of every state agg: a non-NULL row count that disagrees with pass 1's is an error.
__global__ void k_state_check(const uint64_t *state, const StateCol *scols, const StateArgs A) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < A.n_segs; i += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t g = i / A.n_cells, cell = i - g * A.n_cells;
    if (A.rows[i] != state[scols[g].count_off + cell]) gauge_mismatch(A.status, A.err_page);
  }
}

// The state agg outputs (blockIdx.y: the state agg; output column out0 + blockIdx.y): the cell's map entries (u64,
// always valid).
__global__ void k_finalize_states(const StateArgs A, uint32_t out0, uint64_t bitmap_stride, uint64_t *values, uint8_t *validity) {
  const uint64_t cell = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const bool valid = cell < A.n_cells;
  if (valid) {
    const uint64_t s = (uint64_t)blockIdx.y * A.n_cells + cell;
    values[(uint64_t)(out0 + blockIdx.y) * A.n_cells + cell] = (uint64_t)(A.off[s + 1] - A.off[s]);
  }
  const uint32_t bits = __ballot_sync(FULL, valid);
  if ((threadIdx.x & 31) == 0 && (cell >> 3) < bitmap_stride)
    *reinterpret_cast<uint32_t *>(validity + (uint64_t)(out0 + blockIdx.y) * bitmap_stride + (cell >> 3)) = bits;
}

// ---- state periods (TSKV_STATE_PERIODS): state_agg(time, x)'s periods, for state_at and duration_in with a start --------
// The duration records tile every series' timeline from its first selected point to its last: a run record [t0, t'),
// a piece's open run [t0, last t) and a stitch record [last t, next piece's first t), each of the state at its start.
// After the stitch (before the duration sorts, which overwrite the segments), a stable sort by start time and the stable
// sorts by state key and by segment order the records by (segment, key, start); a record of length 0, of an operand
// without the flag or past the last record gets the segment ~0 and sorts last. A record whose predecessor has the same
// segment and key and ends where it starts joins the predecessor's period (the reference's periods of one pair of points
// each, joined where they touch); the others start a period. An exclusive sum over the period heads gives every record
// its period, the heads write the starts and the last record of a period its end. The output order is the CSR order.
struct PeriodArgs {
  uint64_t *pkey;   // [2 * dbound] sort keys: start time keys | sorted, then state keys | sorted, then segments | sorted
  uint32_t *idx;    // [2 * dbound] positions: identity | time order | (time, key) order | (segment, key, start) order
  uint32_t *head;   // [dbound + 1] 1: the record in (segment, key, start) order starts a period
  uint32_t *pos;    // [dbound + 1] the heads' exclusive sum (pos[dbound]: the periods)
  StateKey *out_key;  // [dbound] each period's segment and state key
  int64_t *out_start, *out_end;  // [dbound] each period's start and end
  uint32_t *off;    // [n_segs + 1] the periods per (agg, cell), then their exclusive sum (the CSR offsets)
  uint32_t agg_mask;  // bit g: state agg g has the flag
};

// The records' start time keys (as the boundary records' time keys: start - t_base, clamped to t_mask) and the identity.
__global__ void k_period_keys(const StateArgs A, const PeriodArgs Q) {
  const uint64_t n = min((uint64_t)*A.n_dur, A.dbound);
  for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < A.dbound; j += (uint64_t)gridDim.x * blockDim.x) {
    uint64_t k = 0;
    if (j < n) {
      const int64_t t = A.start[j];
      k = t < A.t_base ? 0 : min((uint64_t)t - (uint64_t)A.t_base, A.t_mask);
    }
    Q.pkey[j] = k;
    Q.idx[j] = (uint32_t)j;
  }
}

// In (time, key) order: the segment a record sorts by (~0: it is no period's part).
__global__ void k_period_segs(const StateArgs A, const PeriodArgs Q) {
  const uint64_t n = min((uint64_t)*A.n_dur, A.dbound);
  for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < A.dbound; j += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t i = Q.idx[j];
    const uint64_t s = A.seg[i];
    const bool keep = i < n && s != ~0ull && A.dur[i] > 0 && ((Q.agg_mask >> ((s >> 1) / A.n_cells)) & 1);
    Q.pkey[j] = keep ? s : ~0ull;
  }
}

// In (segment, key, start) order (segments Q.pkey + dbound, positions Q.idx + dbound): the period heads, counted per
// (agg, cell).
__global__ void k_period_mark(const StateArgs A, const PeriodArgs Q) {
  const uint64_t *seg = Q.pkey + A.dbound;
  const uint32_t *idx = Q.idx + A.dbound;
  for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j <= A.dbound; j += (uint64_t)gridDim.x * blockDim.x) {
    bool h = false;
    if (j < A.dbound && seg[j] != ~0ull) {
      const uint32_t i = idx[j];
      h = true;
      if (j && seg[j - 1] == seg[j]) {
        const uint32_t p = idx[j - 1];
        h = !(A.key[p] == A.key[i] && A.start[p] + A.dur[p] == A.start[i]);
      }
      if (h) atomicAdd(Q.off + (seg[j] >> 1), 1u);
    }
    Q.head[j] = h;
  }
}

// After the heads' exclusive sum: the periods' states, starts and ends.
__global__ void k_period_write(const StateArgs A, const PeriodArgs Q) {
  const uint64_t *seg = Q.pkey + A.dbound;
  const uint32_t *idx = Q.idx + A.dbound;
  for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < A.dbound; j += (uint64_t)gridDim.x * blockDim.x) {
    if (seg[j] == ~0ull) continue;
    const uint32_t i = idx[j], g = Q.pos[j] + Q.head[j] - 1;
    if (Q.head[j]) {
      StateKey k;
      k.seg = seg[j];
      k.key = A.key[i];
      Q.out_key[g] = k;
      Q.out_start[g] = A.start[i];
    }
    if (j + 1 == A.dbound || Q.head[j + 1] || seg[j + 1] == ~0ull) Q.out_end[g] = A.start[i] + A.dur[i];
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
      case TSKV_AGG_M2:
        valid = cnt > 0;
        if (valid) {  // src = sum(d^2), val = sum(d): the corrected two-pass M2 (NaN stays NaN; rounding never goes below 0)
          const double sd = __longlong_as_double((long long)state[oc.val_off + cell]);
          const double m2 = __longlong_as_double((long long)state[oc.src_off + cell]) - sd * sd / (double)cnt;
          v = (uint64_t)__double_as_longlong(m2 < 0.0 ? 0.0 : m2);
        }
        break;
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
