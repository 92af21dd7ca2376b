// tskv_gpu.cu — C-ABI entry points of include/tskv_gpu.h: context, page upload, decode-only and the
// fused scan/aggregate launches. Host logic only; the device code is in scan_kernels.cuh.
#include <algorithm>
#include <cmath>
#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <numeric>
#include <string>
#include <thread>
#include <vector>

#include <cuda_runtime.h>
#include <dlfcn.h>
#include <nccl.h>  // types and enums only: the library is loaded with dlopen on first use

#include "host_util.h"
#include "decode_kernels.cuh"
#include "skip_kernels.cuh"
#include "merge_kernels.cuh"

using namespace tskv;

#define CU_TRY(ctx, expr)                                                              \
  do {                                                                                 \
    cudaError_t e__ = (expr);                                                          \
    if (e__ != cudaSuccess) {                                                          \
      (ctx)->set_error(std::string(#expr) + ": " + cudaGetErrorString(e__));           \
      return e__ == cudaErrorMemoryAllocation ? TSKV_ERR_OOM : TSKV_ERR_CUDA;          \
    }                                                                                  \
  } while (0)

struct tskv_ctx {
  int device = 0;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  cudaStream_t bin_stream[N_BINS] = {nullptr};  // the per-bin fused kernels run concurrently
  cudaStream_t crc_stream = nullptr;            // per-read CRC checks of HBM-resident pages, next to the fused kernels
  int sm_count = 132;
  int max_dyn_smem = 48 * 1024;
  ncclComm_t comm = nullptr;  // tskvgpu_comm_init
  int n_ranks = 1, rank = 0;
  std::mutex mu;
  std::string err;
  int64_t err_page = -1;
  tskv_counters counters{};
  void set_error(const std::string &m, int64_t page = -1) {
    err = m;
    err_page = page;
  }
};

struct tskv_pages {
  tskv_ctx *ctx = nullptr;
  uint8_t *d_arena = nullptr;       // device copy (or, host-resident mode: gather target)
  const uint8_t *h_mapped = nullptr; // host-resident mode: device-visible alias of the caller's arena
  bool verify_on_read = false;       // host-resident + VERIFY_CRC: CRC32 checked on the device on every scan
  uint32_t *d_crc_tables = nullptr;
  void *h_registered = nullptr;      // range this library page-locked (unregistered on destroy)
  uint64_t arena_len = 0;
  tskv_page_desc *d_descs = nullptr;
  std::vector<tskv_page_desc> h_descs;  // with .reserved = DK kind
  uint64_t n_descs = 0;
  uint32_t *d_time_page_of = nullptr;
  uint32_t n_cg = 0;
  uint32_t *d_cg_time_page = nullptr;
  uint32_t *d_cg_series_rank = nullptr;
  uint32_t *d_series_sorted = nullptr;  // the page set's distinct series ids, ascending (rank -> id)
  uint4 *d_item_info = nullptr;         // per item: page, column group, size, column id | type | kind
  uint32_t *d_rank_cg_start = nullptr, *d_rank_cg = nullptr;  // CSR: series rank -> its column groups (arena order)
  uint8_t *d_page_bin = nullptr;        // decode-kind bin of every field page
  mutable int64_t *d_page_stats = nullptr;  // {min key, max key} of every field page (k_page_stats), built on first use
  uint32_t n_items = 0;
  uint32_t *d_item_page = nullptr;
  uint32_t *d_item_cg = nullptr;
  uint32_t h_bin_start[N_BINS + 1]{};
  uint64_t h_bin_bytes[N_BINS]{};    // field-page bytes per bin (orders the PCIe gathers of host-resident scans)
  uint64_t h_bin_rows[N_BINS]{};     // rows of the bin's field pages (serial cost of its chunks)
  uint32_t *d_bin_start = nullptr;
  // tombstones (tskvgpu_pages_set_tombstones); the epoch invalidates scans prepared before a change
  uint64_t *d_tomb_keys = nullptr;
  uint32_t *d_tomb_off = nullptr;
  tskv_time_range *d_tomb_ranges = nullptr;
  uint32_t n_tomb_keys = 0, n_tomb_global = 0, n_tomb_ranges = 0;
  uint64_t tomb_epoch = 0;
  std::vector<uint32_t> series;  // sorted distinct ids
  // arena-wide time bounds, computed on first use by k_time_bounds (the reference keeps them in
  // PageMeta.statistics); only unbucketed first/last across series needs them
  mutable bool bounds_known = false;
  mutable int64_t ts_min = INT64_MIN, ts_max = INT64_MAX;
  // per-column-group [min_ts, max_ts] (ColumnGroup::time_range()): handed in by the caller
  // (tskvgpu_pages_set_time_bounds) or computed together with the arena-wide bounds; drives statistics pruning
  mutable tskv_time_range *d_cg_bounds = nullptr;
  // row-filter masks: 32-bit words per column group, offset stored at the index of the group's time page
  uint32_t *d_keep_off = nullptr;
  uint64_t keep_words = 0;
  // restart points (skip_kernels.cuh): per page the index of its first entry (or SKIP_NONE), built once at upload
  uint32_t *d_skip_off = nullptr;
  SkipEntry *d_skip = nullptr;
  uint64_t n_skip = 0;
  // per page 1 = a simple8b integer page whose values all lie in [-2^31, 2^31) (i64) / [0, 2^31) (u64) (k_build_skip;
  // null for host-resident page sets: every page is then wide), and per bin whether none, some or all of its pages are
  // narrow (NARROW_*: which variant of the fused kernel runs the bin)
  uint8_t *d_narrow = nullptr;
  uint8_t h_bin_narrow[N_BINS]{};
  uint32_t h_bin_maxrows[N_BINS]{};  // longest field page of each bin (parts per page when a scan cuts the bin's pages)
  // overlapping chunks (tskvgpu_pages_set_chunk_files, merge_kernels.cuh): the plan, its device copies and the merge
  // rows' timestamps (decoded once); the epoch invalidates scans prepared before a change
  std::vector<uint32_t> h_cg_time_page, h_cg_series;
  std::vector<uint8_t> h_time_has_nulls;
  OverlapPlan overlap;
  std::vector<tskv_time_range> h_cg_bounds;
  uint8_t *d_cg_merge = nullptr;
  int64_t *d_merge_ts = nullptr;
  uint64_t *d_mcg_row0 = nullptr, *d_mcg_bm0 = nullptr;
  uint32_t *d_mcg_cg = nullptr, *d_mcg_stream = nullptr, *d_stream_group = nullptr, *d_stream_first_mcg = nullptr,
           *d_group_first_stream = nullptr;
  std::vector<uint64_t> h_mcg_bm0;
  uint64_t merge_rows = 0, merge_bm_words = 0;
  uint64_t chunk_epoch = 0;
};

struct tskv_scan {
  const tskv_pages *pages = nullptr;
  uint64_t tomb_epoch = 0;
  tskv_output_layout layout{};
  StateLayout sl{};
  ScanParams params{};
  uint32_t n_cols = 0, n_out = 0;
  bool has_sel = false;  // any FIRST/LAST
  // device buffers
  uint32_t *d_series = nullptr;
  int32_t *d_rank_slot = nullptr;  // rank of a series in the page set -> position in the selection list (or -1)
  uint32_t *d_bucket = nullptr;    // selection-driven work list: [N_BINS * n_cols * WL_SUB] counts / cursors | [.. + 1] offsets
  bool worklist_by_items = false;  // TSKV_WORKLIST=items: the round-1 pass over every field page of the page set
  int32_t *d_cg_slot = nullptr;
  uint8_t *d_item_flag = nullptr;
  uint32_t *d_block_count = nullptr;
  uint32_t n_blocks = 0;
  uint32_t *d_work_page = nullptr, *d_work_slot = nullptr;
  uint8_t *d_work_qcol = nullptr;
  uint32_t *d_bin_cstart = nullptr;  // [N_BINS+1] then [1] total
  ColState *d_cols = nullptr;
  OutCol *d_outs = nullptr;
  MeanExport *d_means = nullptr;
  uint32_t n_means = 0;
  uint64_t *d_state = nullptr;
  uint32_t *d_task_counter = nullptr;
  int32_t *d_status = nullptr;
  unsigned long long *d_err_page = nullptr;
  unsigned long long *d_stats = nullptr;     // [0] points [1] rows in range
  unsigned long long *d_counters = nullptr;  // [0] pages [1] bytes
  uint64_t *d_values = nullptr;
  uint8_t *d_validity = nullptr;
  int grid[N_BINS] = {0};
  int occ[N_BINS] = {0};  // resident CTAs per SM of each bin's kernel at this scan's shared memory size
  tskv_ctx *ctx = nullptr;
  uint32_t n_series_sel = 0;
  bool enqueued = false;
  // timing / ordering events of THIS scan (several scans of one context may be in flight from different host threads)
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  cudaEvent_t ev_bin[N_BINS + 1] = {nullptr};  // [0] fork, [N_BINS] join of the fused phase
  cudaEvent_t ev_bin_start[N_BINS] = {nullptr}, ev_bin_done[N_BINS] = {nullptr}, ev_gather[N_BINS] = {nullptr};
  tskv_counters counters{};  // of the last completed pass of this scan
  // A scan that is enqueued repeatedly replays its whole pass (2 memsets, ~7 small kernels, the fused kernels forked
  // over the bin streams, export) as ONE CUDA graph launch: captured on the second enqueue, so one-shot scans never pay
  // for a capture.
  cudaGraphExec_t graph_exec = nullptr;
  cudaEvent_t ev_cfork = nullptr, ev_cjoin[N_BINS] = {nullptr};  // dependency-only events of the captured pass
  cudaEvent_t ev_crc = nullptr, ev_ccrc = nullptr;  // join of the concurrent CRC checks (plain / captured pass)
  int32_t *d_crc_status = nullptr;                  // a CRC mismatch outranks whatever the decoders made of the bad page
  unsigned long long *d_crc_err_page = nullptr;
  uint32_t n_enqueued = 0;
  bool graph_failed = false;
  PruneRanges prune{};
  uint64_t *d_gathered = nullptr;  // all ranks' exchange regions (tskvgpu_scan_exchange)
  PredicateSet preds{};            // pushed field predicates (row filter)
  uint32_t *d_row_keep = nullptr;  // one keep bit per row of every column group (k_row_filter)
  // merge pass over the overlapping chunks this scan reads (merge_kernels.cuh)
  uint64_t chunk_epoch = 0;
  MergeParams merge{};
  uint32_t n_merge_pages = 0;      // field pages decoded per pass
  uint64_t merge_page_bytes = 0, merge_read_pages = 0;
  uint8_t *d_mcg_active = nullptr;
  uint64_t *d_mvals = nullptr;
  uint32_t *d_mvalid = nullptr;
  uint32_t *d_mpage = nullptr;
  uint64_t *d_mrow_off = nullptr, *d_mbm_off = nullptr;
  // Layout of the state the fused kernels write at params.state: d_state / sl for a tumbling scan. A sliding scan's
  // kernels fill d_pane_state (panes one slide wide) and k_window_combine folds every run of win_k panes into the
  // windows of d_state / sl, which export, exchange, partials and finalize see.
  StateLayout kern_sl{};
  uint64_t *d_pane_state = nullptr;
  CombineOp *d_combine = nullptr;
  uint32_t n_combine = 0, win_k = 1, n_panes = 0, n_windows = 0;
  // GROUP BY tags: the group of every slot (params.slot_group) and the work-list walk order, slots sorted by group (null
  // when that is the selection order)
  uint32_t *d_slot_group = nullptr, *d_walk = nullptr;
};

namespace {

const char *status_text(tskv_status st) {
  switch (st) {
    case TSKV_OK: return "ok";
    case TSKV_ERR_INVALID_ARG: return "invalid argument";
    case TSKV_ERR_BAD_ENCODING: return "invalid block encoding";
    case TSKV_ERR_SHORT_BLOCK: return "not enough data to decode / unexpected end of block";
    case TSKV_ERR_CRC_MISMATCH: return "TsmPageFileHashCheckFailed: page crc32 mismatch";
    case TSKV_ERR_BITSET_MISMATCH: return "Mismatch between bit set and decoded values";
    case TSKV_ERR_UNSUPPORTED: return "unsupported encoding or query shape";
    case TSKV_ERR_BUCKET_RANGE: return "row outside the requested bucket range";
    case TSKV_ERR_CUDA: return "CUDA error";
    case TSKV_ERR_OOM: return "out of device memory";
    case TSKV_ERR_BAD_LENGTH: return "invalid uncompressed block length";
    case TSKV_ERR_PAGE_FORMAT: return "page shorter than its header/bitset";
    default: return "error";
  }
}

template <typename T>
cudaError_t dev_alloc(T **p, size_t n) {
  return cudaMalloc(reinterpret_cast<void **>(p), std::max<size_t>(n, 1) * sizeof(T));
}

unsigned bits_for(uint64_t max_value) {  // bits needed to represent values in [0, max_value]
  unsigned b = 0;
  while (max_value) {
    b++;
    max_value >>= 1;
  }
  return b;
}

unsigned popc8(unsigned x) { return (unsigned)__builtin_popcount(x & TSKV_AGG_ALL); }

typedef void (*scan_kernel_t)(const ScanParams, int);
// `narrow`: NARROW_* of the bin's pages (tskv_pages::h_bin_narrow); only the simple8b-value kernels without FIRST / LAST
// have narrow variants
template <bool SEL>
scan_kernel_t scan_kernel_for(int bin, int narrow = NARROW_NONE) {
  if constexpr (!SEL) {
    if (narrow == NARROW_SOME && bin == TK_RLE * N_VK + VK_S8B) return k_scan_aggregate<TK_RLE, VK_S8B, false, NARROW_SOME>;
    if (narrow == NARROW_SOME && bin == TK_S8B * N_VK + VK_S8B) return k_scan_aggregate<TK_S8B, VK_S8B, false, NARROW_SOME>;
    if (narrow == NARROW_ALL && bin == TK_RLE * N_VK + VK_S8B) return k_scan_aggregate<TK_RLE, VK_S8B, false, NARROW_ALL>;
    if (narrow == NARROW_ALL && bin == TK_S8B * N_VK + VK_S8B) return k_scan_aggregate<TK_S8B, VK_S8B, false, NARROW_ALL>;
  }
  switch (bin) {
    case TK_RLE * N_VK + VK_S8B: return k_scan_aggregate<TK_RLE, VK_S8B, SEL, NARROW_NONE>;
    case TK_RLE * N_VK + VK_GOR: return k_scan_aggregate<TK_RLE, VK_GOR, SEL, NARROW_NONE>;
    case TK_RLE * N_VK + VK_GEN: return k_scan_aggregate<TK_RLE, VK_GEN, SEL, NARROW_NONE>;
    case TK_S8B * N_VK + VK_S8B: return k_scan_aggregate<TK_S8B, VK_S8B, SEL, NARROW_NONE>;
    case TK_S8B * N_VK + VK_GOR: return k_scan_aggregate<TK_S8B, VK_GOR, SEL, NARROW_NONE>;
    case TK_S8B * N_VK + VK_GEN: return k_scan_aggregate<TK_S8B, VK_GEN, SEL, NARROW_NONE>;
    case TK_GEN * N_VK + VK_S8B: return k_scan_aggregate<TK_GEN, VK_S8B, SEL, NARROW_NONE>;
    case TK_GEN * N_VK + VK_GOR: return k_scan_aggregate<TK_GEN, VK_GOR, SEL, NARROW_NONE>;
    default: return k_scan_aggregate<TK_GEN, VK_GEN, SEL, NARROW_NONE>;
  }
}
// the bin among 0-8 whose lane-per-page kernel also runs a short-page bin
int serial_bin_of(int bin) {
  if (bin == BIN_SHORT_RLE_S8B) return TK_RLE * N_VK + VK_S8B;
  if (bin == BIN_SHORT_S8B_S8B) return TK_S8B * N_VK + VK_S8B;
  if (bin == BIN_SHORT_RLE_GOR) return TK_RLE * N_VK + VK_GOR;
  if (bin == BIN_SHORT_S8B_GOR) return TK_S8B * N_VK + VK_GOR;
  return bin;
}

// dynamic shared memory of a lane-per-page kernel: the per-CTA table + the warps' staging rings and flush areas + the
// lanes' tombstone lists when the page set has tombstones
size_t serial_smem_bytes(int serial_bin, uint32_t table_words, bool has_tomb) {
  return (size_t)((table_words + 1) & ~1u) * 8 + (size_t)scan_warp_bytes(serial_bin / N_VK) * (SCAN_THREADS / 32) +
         (has_tomb ? SCAN_TOMB_BYTES : 0);
}
// Serial time of one row of one 32-page chunk, relative: simple8b timestamps cost more than RLE ones (closed form),
// gorilla values more than simple8b ones, generic codecs most. Only the order and rough ratios matter: they rank the
// bin streams' priorities and weigh the bins in plan_serial_grids.
double chunk_cost(int bin) {
  static const double tk[N_TK] = {0.0, 0.16, 0.35}, vk[N_VK] = {0.28, 0.31, 0.45};
  const int sb = serial_bin_of(bin);
  return tk[sb / N_VK] + vk[sb % N_VK];
}

// Lazily computes the arena's min / max timestamp on the device (one lane per time page).
void ensure_time_bounds(tskv_ctx *ctx, const tskv_pages *pg) {
  if (pg->bounds_known || pg->n_cg == 0) return;
  long long *d_bounds = nullptr;
  if (cudaMalloc(reinterpret_cast<void **>(&d_bounds), 16) != cudaSuccess) return;
  long long b[2] = {INT64_MAX, INT64_MIN};
  cudaMemcpyAsync(d_bounds, b, sizeof(b), cudaMemcpyHostToDevice, ctx->stream);
  if (!pg->d_cg_bounds && cudaMalloc(reinterpret_cast<void **>(&pg->d_cg_bounds), (size_t)pg->n_cg * sizeof(tskv_time_range)) != cudaSuccess)
    pg->d_cg_bounds = nullptr;
  k_time_bounds<<<(pg->n_cg + 127) / 128, 128, 0, ctx->stream>>>(pg->h_mapped ? pg->h_mapped : pg->d_arena, pg->d_descs,
                                                                pg->d_cg_time_page, pg->n_cg, d_bounds, pg->d_cg_bounds);
  if (cudaMemcpyAsync(b, d_bounds, sizeof(b), cudaMemcpyDeviceToHost, ctx->stream) == cudaSuccess &&
      cudaStreamSynchronize(ctx->stream) == cudaSuccess && b[0] <= b[1]) {
    pg->ts_min = b[0];
    pg->ts_max = b[1];
  }
  pg->bounds_known = true;
  cudaFree(d_bounds);
}

// Value statistics of the field pages, computed on the device the first time a scan with field predicates is prepared
// (pages resident in HBM only; the reference reads them from PageMeta.statistics).
void ensure_page_stats(tskv_ctx *ctx, const tskv_pages *pg) {
  static const bool off = getenv("TSKV_NO_VALUE_STATS") != nullptr;
  if (off || pg->d_page_stats || pg->h_mapped || pg->n_descs == 0) return;
  int64_t *d = nullptr;
  if (cudaMalloc(reinterpret_cast<void **>(&d), (size_t)pg->n_descs * 16) != cudaSuccess) {
    cudaGetLastError();
    return;
  }
  k_page_stats<<<(unsigned)((pg->n_descs + 127) / 128), 128, 0, ctx->stream>>>(pg->d_arena, pg->d_descs, pg->n_descs, d);
  if (cudaGetLastError() != cudaSuccess || cudaStreamSynchronize(ctx->stream) != cudaSuccess) {
    cudaFree(d);
    return;
  }
  pg->d_page_stats = d;
}

// GROUP BY tags (the *_grouped entry points): group of every selected series slot, and the number of groups.
struct TagGroups {
  bool on = false;
  const uint32_t *ids = nullptr;
  uint32_t n = 0;
};

uint64_t selected_slots(const tskv_pages *pages, const tskv_query *q) { return q->series_ids ? q->n_series : pages->series.size(); }

// Why a group map is refused (TSKV_ERR_INVALID_ARG), or null.
const char *tag_groups_refusal(const tskv_pages *pages, const tskv_query *q, const TagGroups &tg) {
  if (!tg.on) return nullptr;
  if (!tg.ids || tg.n == 0) return "GROUP BY tags: group_ids must be non-null and n_groups >= 1";
  if (q->group_by_series) return "GROUP BY tags: group_by_series must be 0 (the group map replaces it)";
  if ((uint64_t)tg.n * q->n_buckets > TSKV_MAX_GROUPED_CELLS) return "GROUP BY tags: n_groups x n_buckets exceeds TSKV_MAX_GROUPED_CELLS";
  const uint64_t n_slots = selected_slots(pages, q);
  for (uint64_t i = 0; i < n_slots; i++)
    if (tg.ids[i] >= tg.n) return "GROUP BY tags: a group id is >= n_groups";
  return nullptr;
}

tskv_status compute_layout(const tskv_pages *pages, const tskv_query *q, const TagGroups &tg, tskv_output_layout *out) {
  if (!pages || !q || !out || q->n_buckets == 0 || q->n_columns == 0 || !q->columns) return TSKV_ERR_INVALID_ARG;
  if (q->width <= 0 && q->n_buckets != 1) return TSKV_ERR_INVALID_ARG;
  if (tag_groups_refusal(pages, q, tg)) return TSKV_ERR_INVALID_ARG;
  uint64_t n_out = 0;
  for (uint32_t c = 0; c < q->n_columns; c++) n_out += popc8(q->columns[c].agg_mask);
  uint64_t n_groups = 1;
  if (q->group_by_series) n_groups = selected_slots(pages, q);
  if (tg.on) n_groups = tg.n;
  out->n_out = n_out;
  out->n_groups = n_groups;
  out->n_cells = n_groups * q->n_buckets;
  out->bitmap_stride = (out->n_cells + 63) / 64 * 8;
  out->values_bytes = n_out * out->n_cells * 8;
  out->validity_bytes = n_out * out->bitmap_stride;
  return TSKV_OK;
}

// Offsets of the partial state of `q` over n_cells cells: the sections tskv_partials_view exposes, in that order, then
// the scan's own arrays (first / last pairs, key snapshot, high words of exact integer sums).
struct StatePlan {
  StateLayout sl{};
  std::vector<ColState> cols;
  std::vector<MeanExport> means;
  std::vector<uint64_t> msum_off;  // per column: the exported f64 exact integer sum of MEAN, or 0
};
StatePlan plan_state(const tskv_query *q, uint64_t n_cells) {
  StatePlan plan;
  plan.cols.resize(q->n_columns);
  plan.msum_off.assign(q->n_columns, 0);
  std::vector<ColState> &cols = plan.cols;
  std::vector<MeanExport> &means = plan.means;
  std::vector<uint64_t> &msum_off = plan.msum_off;
  StateLayout &sl = plan.sl;
  uint64_t off = 0;
  sl.sum_i64_off = off;
  for (uint32_t c = 0; c < q->n_columns; c++) {
    const tskv_agg_column &qc = q->columns[c];
    cols[c] = ColState{};
    cols[c].column_id = qc.column_id;
    cols[c].phys_type = qc.phys_type;
    cols[c].agg_mask = qc.agg_mask;
    cols[c].count_off = off;
    off += n_cells;
    if ((qc.agg_mask & (TSKV_AGG_SUM | TSKV_AGG_MEAN)) && qc.phys_type != TSKV_PT_F64) {
      cols[c].sum_off = off;
      off += n_cells;
    }
  }
  sl.sum_i64_len = off - sl.sum_i64_off;
  sl.sum_f64_off = off;
  for (uint32_t c = 0; c < q->n_columns; c++)
    if ((q->columns[c].agg_mask & (TSKV_AGG_SUM | TSKV_AGG_MEAN)) && q->columns[c].phys_type == TSKV_PT_F64) {
      cols[c].sum_off = off;
      off += n_cells;
    }
  for (uint32_t c = 0; c < q->n_columns; c++)
    if ((q->columns[c].agg_mask & TSKV_AGG_MEAN) && q->columns[c].phys_type != TSKV_PT_F64) {
      msum_off[c] = off;  // exported exact integer sum as f64 (all-reducible)
      off += n_cells;
    }
  sl.sum_f64_len = off - sl.sum_f64_off;
  uint64_t n_first = 0, n_last = 0;
  for (uint32_t c = 0; c < q->n_columns; c++) {
    if (q->columns[c].agg_mask & TSKV_AGG_FIRST) n_first += n_cells;
    if (q->columns[c].agg_mask & TSKV_AGG_LAST) n_last += n_cells;
  }
  sl.first_cells = n_first;
  sl.last_cells = n_last;
  sl.min_off = off;
  for (uint32_t c = 0; c < q->n_columns; c++)
    if (q->columns[c].agg_mask & TSKV_AGG_MIN) {
      cols[c].min_off = off;
      off += n_cells;
    }
  sl.first_keys_off = off;
  off += n_first;
  sl.min_len = off - sl.min_off;
  sl.max_off = off;
  for (uint32_t c = 0; c < q->n_columns; c++)
    if (q->columns[c].agg_mask & TSKV_AGG_MAX) {
      cols[c].max_off = off;
      off += n_cells;
    }
  sl.last_keys_off = off;
  off += n_last;
  sl.max_len = off - sl.max_off;
  sl.selval_off = off;
  off += n_first + n_last;
  sl.selval_len = n_first + n_last;
  off = (off + 1) & ~1ull;  // 16-byte alignment of the pair arrays
  sl.first_pairs_off = off;
  {
    uint64_t o = off;
    for (uint32_t c = 0; c < q->n_columns; c++)
      if (q->columns[c].agg_mask & TSKV_AGG_FIRST) {
        cols[c].first_off = o;
        o += 2 * n_cells;
      }
    off = o;
  }
  sl.last_pairs_off = off;
  {
    uint64_t o = off;
    for (uint32_t c = 0; c < q->n_columns; c++)
      if (q->columns[c].agg_mask & TSKV_AGG_LAST) {
        cols[c].last_off = o;
        o += 2 * n_cells;
      }
    off = o;
  }
  sl.snap_off = off;
  off += n_first + n_last;
  for (uint32_t c = 0; c < q->n_columns; c++)
    if (msum_off[c]) {
      cols[c].sumhi_off = off;
      means.push_back(MeanExport{cols[c].sum_off, off, msum_off[c], q->columns[c].phys_type == TSKV_PT_I64 ? 1u : 0u, 0});
      off += n_cells;
    }
  sl.total = off;
  return plan;
}

// Per-scan buffers are stream-ordered (cudaMallocAsync on the context stream): no device-wide
// synchronisation on the query path, memory is recycled by the pool.
void free_scan(tskv_scan *s) {
  if (!s) return;
  cudaStream_t st = s->ctx ? s->ctx->stream : nullptr;
  void *bufs[] = {s->d_series, s->d_rank_slot, s->d_bucket, s->d_cg_slot, s->d_item_flag, s->d_block_count, s->d_work_page, s->d_work_slot,
                  s->d_work_qcol, s->d_bin_cstart, s->d_cols, s->d_outs, s->d_means, s->d_state,
                  s->d_task_counter, s->d_values, s->d_validity, s->d_gathered, s->d_row_keep,
                  s->d_mcg_active, s->d_mvals, s->d_mvalid, s->d_mpage, s->d_mrow_off, s->d_mbm_off, s->d_pane_state, s->d_combine,
                  s->d_slot_group, s->d_walk};
  for (void *b : bufs)
    if (b) cudaFreeAsync(b, st);
  if (s->graph_exec) cudaGraphExecDestroy(s->graph_exec);
  if (s->ev_cfork) cudaEventDestroy(s->ev_cfork);
  if (s->ev_crc) cudaEventDestroy(s->ev_crc);
  if (s->ev_ccrc) cudaEventDestroy(s->ev_ccrc);
  for (int b = 0; b < N_BINS; b++)
    if (s->ev_cjoin[b]) cudaEventDestroy(s->ev_cjoin[b]);
  if (s->ev0) cudaEventDestroy(s->ev0);
  if (s->ev1) cudaEventDestroy(s->ev1);
  for (int b = 0; b <= N_BINS; b++)
    if (s->ev_bin[b]) cudaEventDestroy(s->ev_bin[b]);
  for (int b = 0; b < N_BINS; b++) {
    if (s->ev_bin_start[b]) cudaEventDestroy(s->ev_bin_start[b]);
    if (s->ev_bin_done[b]) cudaEventDestroy(s->ev_bin_done[b]);
    if (s->ev_gather[b]) cudaEventDestroy(s->ev_gather[b]);
  }
  delete s;
}

void free_overlap(tskv_pages *pg) {
  void *bufs[] = {pg->d_cg_merge, pg->d_merge_ts, pg->d_mcg_row0, pg->d_mcg_bm0, pg->d_mcg_cg, pg->d_mcg_stream,
                  pg->d_stream_group, pg->d_stream_first_mcg, pg->d_group_first_stream};
  for (void *b : bufs) cudaFree(b);
  pg->d_cg_merge = nullptr; pg->d_merge_ts = nullptr; pg->d_mcg_row0 = nullptr; pg->d_mcg_bm0 = nullptr; pg->d_mcg_cg = nullptr;
  pg->d_mcg_stream = nullptr; pg->d_stream_group = nullptr; pg->d_stream_first_mcg = nullptr; pg->d_group_first_stream = nullptr;
  pg->overlap = OverlapPlan{};
  pg->merge_rows = pg->merge_bm_words = 0;
  pg->h_mcg_bm0.clear();
}

template <typename T>
cudaError_t stream_alloc(tskv_ctx *ctx, T **p, size_t n) {
  return cudaMallocAsync(reinterpret_cast<void **>(p), std::max<size_t>(n, 1) * sizeof(T), ctx->stream);
}

// Reads back the device status word; maps it to a message.
tskv_status fetch_status(tskv_ctx *ctx, int32_t *d_status, unsigned long long *d_err_page) {
  int32_t st = 0;
  unsigned long long pg = 0;
  if (cudaMemcpyAsync(&st, d_status, sizeof(st), cudaMemcpyDeviceToHost, ctx->stream) != cudaSuccess ||
      cudaMemcpyAsync(&pg, d_err_page, sizeof(pg), cudaMemcpyDeviceToHost, ctx->stream) != cudaSuccess ||
      cudaStreamSynchronize(ctx->stream) != cudaSuccess) {
    ctx->set_error(std::string("status readback: ") + cudaGetErrorString(cudaGetLastError()));
    return TSKV_ERR_CUDA;
  }
  if (st != TSKV_OK) ctx->set_error(std::string(status_text(st)) + " (page " + std::to_string(pg) + ")", (int64_t)pg);
  return st;
}

// NCCL entry points, resolved from libnccl.so.2 on first use.
struct NcclApi {
  ncclResult_t (*GetUniqueId)(ncclUniqueId *) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t *, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*AllGather)(const void *, void *, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
  const char *(*GetErrorString)(ncclResult_t) = nullptr;
  bool ok = false;
};
const NcclApi &nccl_api() {
  static NcclApi api;
  static std::once_flag once;
  std::call_once(once, []() {
    void *h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
    if (!h) return;
    api.GetUniqueId = reinterpret_cast<decltype(api.GetUniqueId)>(dlsym(h, "ncclGetUniqueId"));
    api.CommInitRank = reinterpret_cast<decltype(api.CommInitRank)>(dlsym(h, "ncclCommInitRank"));
    api.CommDestroy = reinterpret_cast<decltype(api.CommDestroy)>(dlsym(h, "ncclCommDestroy"));
    api.AllGather = reinterpret_cast<decltype(api.AllGather)>(dlsym(h, "ncclAllGather"));
    api.GetErrorString = reinterpret_cast<decltype(api.GetErrorString)>(dlsym(h, "ncclGetErrorString"));
    api.ok = api.GetUniqueId && api.CommInitRank && api.CommDestroy && api.AllGather && api.GetErrorString;
  });
  return api;
}

}  // namespace

extern "C" {

static_assert(sizeof(ncclUniqueId) == TSKV_NCCL_UNIQUE_ID_BYTES, "tskv_gpu.h: NCCL unique id size");

tskv_status tskvgpu_comm_unique_id(uint8_t *out_id) {
  const NcclApi &N = nccl_api();
  if (!out_id) return TSKV_ERR_INVALID_ARG;
  if (!N.ok) return TSKV_ERR_NCCL;
  ncclUniqueId id;
  if (N.GetUniqueId(&id) != ncclSuccess) return TSKV_ERR_NCCL;
  memcpy(out_id, &id, sizeof(id));
  return TSKV_OK;
}

tskv_status tskvgpu_comm_init(tskv_ctx *ctx, const uint8_t *id_bytes, int32_t rank, int32_t n_ranks) {
  if (!ctx || !id_bytes || n_ranks < 1 || rank < 0 || rank >= n_ranks) return TSKV_ERR_INVALID_ARG;
  const NcclApi &N = nccl_api();
  std::lock_guard<std::mutex> lock(ctx->mu);
  ctx->set_error("");
  if (!N.ok) {
    ctx->set_error("libnccl.so.2 could not be loaded");
    return TSKV_ERR_NCCL;
  }
  CU_TRY(ctx, cudaSetDevice(ctx->device));
  if (ctx->comm) {
    N.CommDestroy(ctx->comm);
    ctx->comm = nullptr;
  }
  ncclUniqueId id;
  memcpy(&id, id_bytes, sizeof(id));
  const ncclResult_t r = N.CommInitRank(&ctx->comm, n_ranks, id, rank);
  if (r != ncclSuccess) {
    ctx->set_error(std::string("ncclCommInitRank: ") + N.GetErrorString(r));
    ctx->comm = nullptr;
    return TSKV_ERR_NCCL;
  }
  ctx->n_ranks = n_ranks;
  ctx->rank = rank;
  return TSKV_OK;
}

void tskvgpu_comm_destroy(tskv_ctx *ctx) {
  if (!ctx || !ctx->comm) return;
  std::lock_guard<std::mutex> lock(ctx->mu);
  cudaSetDevice(ctx->device);
  cudaStreamSynchronize(ctx->stream);
  nccl_api().CommDestroy(ctx->comm);
  ctx->comm = nullptr;
  ctx->n_ranks = 1;
}

const char *tskvgpu_version(void) { return "tskv-b200 0.1.0 sm_90a"; }

tskv_status tskvgpu_ctx_create(int32_t device_id, tskv_ctx **out_ctx) {
  if (!out_ctx) return TSKV_ERR_INVALID_ARG;
  *out_ctx = nullptr;
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || device_id < 0 || device_id >= n) return TSKV_ERR_CUDA;
  tskv_ctx *ctx = new tskv_ctx();
  ctx->device = device_id;
  if (cudaSetDevice(device_id) != cudaSuccess ||
      cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking) != cudaSuccess ||
      cudaEventCreate(&ctx->ev0) != cudaSuccess || cudaEventCreate(&ctx->ev1) != cudaSuccess) {
    delete ctx;
    return TSKV_ERR_CUDA;
  }
  cudaDeviceGetAttribute(&ctx->sm_count, cudaDevAttrMultiProcessorCount, device_id);
  {
    // Bins whose chunks take longest get the highest stream priority: when the grids of a scan over-subscribe the
    // machine, the block scheduler starts the long serial tasks first and back-fills with the short ones.
    int least = 0, greatest = 0;
    cudaDeviceGetStreamPriorityRange(&least, &greatest);
    for (int b = 0; b < N_BINS; b++) {
      int rank = 0;
      for (int o = 0; o < N_BINS; o++) rank += chunk_cost(o) > chunk_cost(b) ? 1 : 0;
      const int prio = std::min(least, greatest + rank / 2);
      if (cudaStreamCreateWithPriority(&ctx->bin_stream[b], cudaStreamNonBlocking, prio) != cudaSuccess)
        cudaStreamCreateWithFlags(&ctx->bin_stream[b], cudaStreamNonBlocking);
    }
    // (TSKV_CRC_CONCURRENT: the per-read CRC checks on a stream of their own)
    if (cudaStreamCreateWithPriority(&ctx->crc_stream, cudaStreamNonBlocking, greatest) != cudaSuccess)
      cudaStreamCreateWithFlags(&ctx->crc_stream, cudaStreamNonBlocking);
  }
  // Dynamic shared memory ceiling of every scan kernel, set ONCE: the attribute belongs to the kernel, not to a launch,
  // so per-scan values would race between host threads that prepare scans with different table sizes.
  {
    int optin = 0;
    cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device_id);
    ctx->max_dyn_smem = optin;
    auto raise = [&](const void *fn) {  // the opt-in limit covers static + dynamic shared memory
      cudaFuncAttributes fa{};
      if (cudaFuncGetAttributes(&fa, fn) == cudaSuccess)
        cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, optin - (int)fa.sharedSizeBytes);
    };
    for (int b = 0; b < N_SERIAL_BINS; b++) {
      for (int nm = NARROW_NONE; nm <= NARROW_ALL; nm++) raise((const void *)scan_kernel_for<false>(b, nm));
      raise((const void *)scan_kernel_for<true>(b));
    }
    cudaGetLastError();
  }
  // per-scan buffers come from the stream-ordered pool; keep freed memory cached in the pool
  cudaMemPool_t pool;
  if (cudaDeviceGetDefaultMemPool(&pool, device_id) == cudaSuccess) {
    uint64_t thr = UINT64_MAX;
    cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr);
  }
  *out_ctx = ctx;
  return TSKV_OK;
}

void tskvgpu_ctx_destroy(tskv_ctx *ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  if (ctx->comm) tskvgpu_comm_destroy(ctx);
  if (ctx->stream) {
    cudaStreamSynchronize(ctx->stream);
    cudaStreamDestroy(ctx->stream);
  }
  if (ctx->ev0) cudaEventDestroy(ctx->ev0);
  if (ctx->ev1) cudaEventDestroy(ctx->ev1);
  for (int b = 0; b < N_BINS; b++)
    if (ctx->bin_stream[b]) cudaStreamDestroy(ctx->bin_stream[b]);
  if (ctx->crc_stream) cudaStreamDestroy(ctx->crc_stream);
  delete ctx;
}

const char *tskvgpu_last_error(const tskv_ctx *ctx) { return ctx ? ctx->err.c_str() : "null context"; }
int64_t tskvgpu_last_error_page(const tskv_ctx *ctx) { return ctx ? ctx->err_page : -1; }
tskv_status tskvgpu_get_counters(const tskv_ctx *ctx, tskv_counters *out) {
  if (!ctx || !out) return TSKV_ERR_INVALID_ARG;
  *out = ctx->counters;
  return TSKV_OK;
}
uint64_t tskvgpu_ctx_stream(const tskv_ctx *ctx) { return ctx ? (uint64_t)(uintptr_t)ctx->stream : 0; }

// ------------------------------------------------------------------------------------------------
tskv_status tskvgpu_upload_pages(tskv_ctx *ctx, const uint8_t *arena, uint64_t arena_len,
                                 const tskv_page_desc *descs, uint64_t n_descs, uint32_t flags,
                                 tskv_pages **out_pages) {
  if (!ctx || !out_pages || (!arena && arena_len) || (!descs && n_descs)) return TSKV_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(ctx->mu);
  *out_pages = nullptr;
  ctx->set_error("");
  if (n_descs >= (1ull << 32)) {
    ctx->set_error("too many pages for one arena (2^32)");
    return TSKV_ERR_INVALID_ARG;
  }
  cudaSetDevice(ctx->device);
  tskv_pages *pg = new tskv_pages();
  pg->ctx = ctx;
  pg->arena_len = arena_len;
  pg->n_descs = n_descs;
  pg->h_descs.assign(descs, descs + n_descs);

  // ---- framing validation + decode-kind classification (+ CRC), parallel over pages ----------
  std::vector<uint8_t> time_has_nulls(n_descs, 0);
  std::atomic<int> bad_status{0};
  std::atomic<int64_t> bad_page{-1};
  auto fail = [&](int st, int64_t p) {
    int exp = 0;
    if (bad_status.compare_exchange_strong(exp, st)) bad_page = p;
  };
  unsigned hw = std::max(1u, std::min(32u, std::thread::hardware_concurrency()));
  unsigned nthreads = n_descs > 4096 ? hw : 1;
  auto work = [&](uint64_t lo, uint64_t hi) {
    for (uint64_t i = lo; i < hi && bad_status.load(std::memory_order_relaxed) == 0; i++) {
      tskv_page_desc &d = pg->h_descs[i];
      if (d.offset & 15 || d.size > arena_len || d.offset > arena_len - d.size || d.phys_type > TSKV_PT_BOOL || d.reserved != 0) {
        fail(TSKV_ERR_INVALID_ARG, (int64_t)i);
        return;
      }
      PageHeader h;
      if (!parse_page(arena + d.offset, d.size, &h)) {
        d.reserved = DK_BAD_PAGE;
        continue;
      }
      if (h.n_rows != d.num_values) {
        d.reserved = DK_BAD_PAGE;
        continue;
      }
      if ((flags & TSKV_UPLOAD_VERIFY_CRC) && !(flags & TSKV_UPLOAD_HOST_RESIDENT) && crc32_ieee(h.data, h.data_len) != h.crc) {
        fail(TSKV_ERR_CRC_MISMATCH, (int64_t)i);
        return;
      }
      d.reserved = classify_page(h, d.phys_type);
      if (d.phys_type == TSKV_PT_TIME) {  // the fast time cursors assume a time column without nulls
        bool all_valid = true;
        for (uint64_t r = 0; r + 8 <= h.n_rows && all_valid; r += 8) all_valid = h.bitset[r >> 3] == 0xff;
        for (uint64_t r = h.n_rows & ~7ull; r < h.n_rows && all_valid; r++) all_valid = (h.bitset[r >> 3] >> (r & 7)) & 1;
        time_has_nulls[i] = all_valid ? 0 : 1;
      }
    }
  };
  if (nthreads == 1) {
    work(0, n_descs);
  } else {
    std::vector<std::thread> th;
    uint64_t per = (n_descs + nthreads - 1) / nthreads;
    for (unsigned t = 0; t < nthreads; t++) th.emplace_back(work, std::min(n_descs, t * per), std::min(n_descs, (t + 1) * per));
    for (auto &t : th) t.join();
  }
  if (bad_status.load()) {
    tskv_status st = bad_status.load();
    ctx->set_error(st == TSKV_ERR_CRC_MISMATCH ? "TsmPageFileHashCheckFailed: page crc32 mismatch"
                                               : "malformed page descriptor (alignment, bounds, type or reserved != 0)",
                   bad_page.load());
    delete pg;
    return st;
  }

  // ---- column groups, items (field pages) sorted by decode-kind bin ---------------------------
  std::vector<uint32_t> time_page_of(n_descs, 0), cg_time_page, item_page, item_cg;
  {
    uint64_t i = 0;
    while (i < n_descs) {
      if (pg->h_descs[i].phys_type != TSKV_PT_TIME) {
        ctx->set_error("descriptor table: column group does not start with a time page", (int64_t)i);
        delete pg;
        return TSKV_ERR_INVALID_ARG;
      }
      uint32_t cg = (uint32_t)cg_time_page.size();
      cg_time_page.push_back((uint32_t)i);
      time_page_of[i] = (uint32_t)i;
      uint64_t j = i + 1;
      while (j < n_descs && pg->h_descs[j].phys_type != TSKV_PT_TIME) {
        if (pg->h_descs[j].series_id != pg->h_descs[i].series_id || pg->h_descs[j].num_values != pg->h_descs[i].num_values) {
          ctx->set_error("descriptor table: field page disagrees with its time page", (int64_t)j);
          delete pg;
          return TSKV_ERR_INVALID_ARG;
        }
        time_page_of[j] = (uint32_t)i;
        item_page.push_back((uint32_t)j);
        item_cg.push_back(cg);
        j++;
      }
      i = j;
    }
  }
  pg->n_cg = (uint32_t)cg_time_page.size();
  pg->n_items = (uint32_t)item_page.size();
  pg->h_cg_time_page = cg_time_page;
  pg->h_time_has_nulls = time_has_nulls;
  std::vector<uint32_t> keep_off(n_descs, 0);
  for (uint32_t tp : cg_time_page) {
    keep_off[tp] = (uint32_t)pg->keep_words;
    pg->keep_words += ((uint64_t)pg->h_descs[tp].num_values + 31) / 32;
  }
  if (pg->keep_words >= (1ull << 32)) {
    ctx->set_error("too many rows for one arena (2^37)");
    delete pg;
    return TSKV_ERR_INVALID_ARG;
  }
  // series ranks
  pg->series.reserve(pg->n_cg);
  for (uint32_t cg = 0; cg < pg->n_cg; cg++) pg->series.push_back(pg->h_descs[cg_time_page[cg]].series_id);
  std::sort(pg->series.begin(), pg->series.end());
  pg->series.erase(std::unique(pg->series.begin(), pg->series.end()), pg->series.end());
  std::vector<uint32_t> cg_rank(pg->n_cg);
  for (uint32_t cg = 0; cg < pg->n_cg; cg++)
    cg_rank[cg] = (uint32_t)(std::lower_bound(pg->series.begin(), pg->series.end(), pg->h_descs[cg_time_page[cg]].series_id) - pg->series.begin());
  std::vector<uint8_t> page_bin(n_descs, 0);
  // sort items by (bin, column id, arena order): warps are homogeneous in codec and, for GROUP BY
  // bucket, lanes of a warp flush the same (column, bucket) cell in lock step.
  {
    std::vector<uint32_t> order(pg->n_items);
    std::vector<uint64_t> key(pg->n_items);
    for (uint32_t k = 0; k < pg->n_items; k++) {
      const tskv_page_desc &vd = pg->h_descs[item_page[k]];
      const tskv_page_desc &td = pg->h_descs[time_page_of[item_page[k]]];
      int tclass = time_has_nulls[time_page_of[item_page[k]]] ? TK_GEN : time_class(td.reserved);
      uint64_t bin = (uint64_t)tclass * N_VK + value_class(vd.reserved);
      if (vd.num_values <= SHORT_PAGE_ROWS && vd.reserved == DK_S8B_ZZ && tclass != TK_GEN)
        bin = tclass == TK_RLE ? BIN_SHORT_RLE_S8B : BIN_SHORT_S8B_S8B;
      if (vd.num_values <= SHORT_PAGE_ROWS && vd.reserved == DK_GORILLA && tclass != TK_GEN)
        bin = tclass == TK_RLE ? BIN_SHORT_RLE_GOR : BIN_SHORT_S8B_GOR;
      key[k] = (bin << 48) | ((uint64_t)vd.column_id << 32) | k;
      order[k] = k;
      page_bin[item_page[k]] = (uint8_t)bin;
    }
    std::sort(key.begin(), key.end());
    std::vector<uint32_t> ip(pg->n_items), ic(pg->n_items);
    uint32_t counts[N_BINS] = {0};
    for (uint32_t k = 0; k < pg->n_items; k++) {
      uint32_t src = (uint32_t)(key[k] & 0xffffffffu);
      ip[k] = item_page[src];
      ic[k] = item_cg[src];
      counts[key[k] >> 48]++;
      pg->h_bin_bytes[key[k] >> 48] += pg->h_descs[item_page[src]].size;
      pg->h_bin_rows[key[k] >> 48] += pg->h_descs[item_page[src]].num_values;
      pg->h_bin_maxrows[key[k] >> 48] = std::max(pg->h_bin_maxrows[key[k] >> 48], pg->h_descs[item_page[src]].num_values);
    }
    item_page.swap(ip);
    item_cg.swap(ic);
    pg->h_bin_start[0] = 0;
    for (int b = 0; b < N_BINS; b++) pg->h_bin_start[b + 1] = pg->h_bin_start[b] + counts[b];
  }

  // ---- device copies ----------------------------------------------------------------------------
  cudaEventRecord(ctx->ev0, ctx->stream);
  auto up = [&](auto **dptr, const auto *src, size_t n) -> cudaError_t {
    cudaError_t e = dev_alloc(dptr, n);
    if (e != cudaSuccess) return e;
    if (n) e = cudaMemcpyAsync(*dptr, src, n * sizeof(**dptr), cudaMemcpyHostToDevice, ctx->stream);
    return e;
  };
  cudaError_t e = cudaMalloc(reinterpret_cast<void **>(&pg->d_arena), arena_len + ARENA_SLACK);
  if (e == cudaSuccess) e = cudaMemsetAsync(pg->d_arena + arena_len, 0, ARENA_SLACK, ctx->stream);
  if (e == cudaSuccess && arena_len && (flags & TSKV_UPLOAD_HOST_RESIDENT)) {
    // pages stay in (page-locked) host memory like the reference's page cache; each scan pulls the
    // selected pages over PCIe itself (k_gather_pages)
    e = cudaHostRegister(const_cast<uint8_t *>(arena), arena_len, cudaHostRegisterMapped | cudaHostRegisterPortable);
    if (e == cudaSuccess) pg->h_registered = const_cast<uint8_t *>(arena);
    else if (e == cudaErrorHostMemoryAlreadyRegistered) { cudaGetLastError(); e = cudaSuccess; }
    void *dp = nullptr;
    if (e == cudaSuccess) e = cudaHostGetDevicePointer(&dp, const_cast<uint8_t *>(arena), 0);
    pg->h_mapped = static_cast<const uint8_t *>(dp);
  } else if (e == cudaSuccess && arena_len) {
    e = cudaMemcpyAsync(pg->d_arena, arena, arena_len, cudaMemcpyHostToDevice, ctx->stream);
  }
  if (e == cudaSuccess) e = up(&pg->d_descs, pg->h_descs.data(), n_descs);
  if (e == cudaSuccess) e = up(&pg->d_time_page_of, time_page_of.data(), n_descs);
  if (e == cudaSuccess) e = up(&pg->d_cg_time_page, cg_time_page.data(), pg->n_cg);
  if (e == cudaSuccess) e = up(&pg->d_cg_series_rank, cg_rank.data(), pg->n_cg);
  if (e == cudaSuccess) e = up(&pg->d_series_sorted, pg->series.data(), pg->series.size());
  std::vector<uint4> item_info(pg->n_items);
  for (uint32_t k = 0; k < pg->n_items; k++) {
    const tskv_page_desc &d = pg->h_descs[item_page[k]];
    item_info[k] = make_uint4(item_page[k], item_cg[k], d.size, (uint32_t)d.column_id | ((uint32_t)d.phys_type << 16) | ((uint32_t)d.reserved << 24));
  }
  if (e == cudaSuccess) e = up(&pg->d_item_info, item_info.data(), pg->n_items);
  {  // series rank -> its column groups (the selection-driven work list walks a selected series' groups)
    std::vector<uint32_t> start(pg->series.size() + 1, 0), list(pg->n_cg);
    for (uint32_t cg = 0; cg < pg->n_cg; cg++) start[cg_rank[cg] + 1]++;
    for (size_t r = 0; r < pg->series.size(); r++) start[r + 1] += start[r];
    std::vector<uint32_t> cur(start.begin(), start.end() - 1);
    for (uint32_t cg = 0; cg < pg->n_cg; cg++) list[cur[cg_rank[cg]]++] = cg;
    if (e == cudaSuccess) e = up(&pg->d_rank_cg_start, start.data(), start.size());
    if (e == cudaSuccess) e = up(&pg->d_rank_cg, list.data(), list.size());
    if (e == cudaSuccess) e = up(&pg->d_page_bin, page_bin.data(), n_descs);
  }
  if (e == cudaSuccess) e = up(&pg->d_item_page, item_page.data(), pg->n_items);
  if (e == cudaSuccess) e = up(&pg->d_item_cg, item_cg.data(), pg->n_items);
  if (e == cudaSuccess) e = up(&pg->d_bin_start, pg->h_bin_start, N_BINS + 1);
  if (e == cudaSuccess) e = up(&pg->d_keep_off, keep_off.data(), n_descs);
  if (e == cudaSuccess && (((flags & TSKV_UPLOAD_VERIFY_CRC) && (flags & TSKV_UPLOAD_HOST_RESIDENT)) || (flags & TSKV_UPLOAD_VERIFY_ON_READ))) {
    pg->verify_on_read = true;  // like the reference: every read of a page re-checks its CRC (device side)
    e = up(&pg->d_crc_tables, crc32_tables(), 2048);
  }
  // ---- restart points of the simple8b / gorilla pages and narrow flags of the simple8b integer pages (pages resident in
  // HBM only; the flags do not depend on TSKV_NO_SKIP) --------------------------------------------------------------
  const bool no_skip = getenv("TSKV_NO_SKIP") != nullptr;
  if (e == cudaSuccess && !(flags & TSKV_UPLOAD_HOST_RESIDENT) && n_descs) {
    std::vector<uint32_t> skip_off(n_descs, SKIP_NONE), list[3];
    uint64_t n_skip = 0;
    for (uint64_t i = 0; i < n_descs; i++) {
      const tskv_page_desc &d = pg->h_descs[i];
      int kind = -1;
      if (d.phys_type == TSKV_PT_TIME) kind = (d.reserved == DK_S8B_SC && !time_has_nulls[i]) ? SKIP_KIND_TIME_S8B : -1;
      else if (d.reserved == DK_S8B_ZZ) kind = SKIP_KIND_VALUE_S8B;
      else if (d.reserved == DK_GORILLA) kind = SKIP_KIND_VALUE_GORILLA;
      if (kind < 0) continue;
      if (!no_skip && d.num_values > SKIP_ROWS && n_skip + d.num_values / SKIP_ROWS < SKIP_NONE) {
        skip_off[i] = (uint32_t)n_skip;
        n_skip += (d.num_values - 1) / SKIP_ROWS;
      } else if (kind != SKIP_KIND_VALUE_S8B) {
        continue;
      }
      list[kind].push_back((uint32_t)i);
    }
    if (!list[SKIP_KIND_VALUE_S8B].empty()) {
      e = dev_alloc(&pg->d_narrow, n_descs);
      if (e == cudaSuccess) e = cudaMemsetAsync(pg->d_narrow, 0, n_descs, ctx->stream);
    }
    if (n_skip) {
      pg->n_skip = n_skip;
      if (e == cudaSuccess) e = up(&pg->d_skip_off, skip_off.data(), n_descs);
      if (e == cudaSuccess) e = dev_alloc(&pg->d_skip, n_skip);
    }
    const size_t n_list = list[0].size() + list[1].size() + list[2].size();
    if (n_list) {
      uint32_t *d_list = nullptr;
      if (e == cudaSuccess) e = cudaMallocAsync(reinterpret_cast<void **>(&d_list), n_list * 4, ctx->stream);
      size_t lo = 0;
      for (int k = 0; k < 3 && e == cudaSuccess; k++) {
        const uint32_t n = (uint32_t)list[k].size();
        if (!n) continue;
        e = cudaMemcpyAsync(d_list + lo, list[k].data(), (size_t)n * 4, cudaMemcpyHostToDevice, ctx->stream);
        if (e != cudaSuccess) break;
        const uint32_t blocks = (n + SKIP_THREADS - 1) / SKIP_THREADS;
        if (k == SKIP_KIND_TIME_S8B)
          k_build_skip<SKIP_KIND_TIME_S8B><<<blocks, SKIP_THREADS, SKIP_SMEM_BYTES, ctx->stream>>>(pg->d_arena, pg->d_descs, d_list + lo, n, pg->d_skip_off, pg->d_skip, nullptr);
        else if (k == SKIP_KIND_VALUE_S8B)
          k_build_skip<SKIP_KIND_VALUE_S8B><<<blocks, SKIP_THREADS, SKIP_SMEM_BYTES, ctx->stream>>>(pg->d_arena, pg->d_descs, d_list + lo, n, pg->d_skip_off, pg->d_skip, pg->d_narrow);
        else
          k_build_skip<SKIP_KIND_VALUE_GORILLA><<<blocks, SKIP_THREADS, SKIP_SMEM_BYTES, ctx->stream>>>(pg->d_arena, pg->d_descs, d_list + lo, n, pg->d_skip_off, pg->d_skip, nullptr);
        lo += n;
      }
      if (e == cudaSuccess) e = cudaGetLastError();
      // the page lists are read by kernels still in flight: host vectors stay alive until the sync below
      if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
      if (d_list) cudaFreeAsync(d_list, ctx->stream);
    }
    if (e == cudaSuccess && pg->d_narrow) {
      std::vector<uint8_t> narrow(n_descs);
      e = cudaMemcpyAsync(narrow.data(), pg->d_narrow, n_descs, cudaMemcpyDeviceToHost, ctx->stream);
      if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
      uint64_t n_narrow[N_BINS] = {0}, n_pages[N_BINS] = {0};
      for (uint32_t k = 0; k < pg->n_items; k++) {
        n_narrow[page_bin[item_page[k]]] += narrow[item_page[k]];
        n_pages[page_bin[item_page[k]]]++;
      }
      for (int b = 0; b < N_BINS; b++)
        pg->h_bin_narrow[b] = n_narrow[b] == 0 ? NARROW_NONE : n_narrow[b] == n_pages[b] ? NARROW_ALL : NARROW_SOME;
    }
  }
  cudaEventRecord(ctx->ev1, ctx->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
  if (e != cudaSuccess) {
    ctx->set_error(std::string("upload: ") + cudaGetErrorString(e));
    tskvgpu_pages_destroy(nullptr, pg);
    return e == cudaErrorMemoryAllocation ? TSKV_ERR_OOM : TSKV_ERR_CUDA;
  }
  float ms = 0;
  cudaEventElapsedTime(&ms, ctx->ev0, ctx->ev1);
  ctx->counters.elapsed_h2d_ms = ms;
  *out_pages = pg;
  return TSKV_OK;
}

void tskvgpu_pages_destroy(tskv_ctx *ctx, tskv_pages *pg) {
  (void)ctx;
  if (!pg) return;
  if (pg->ctx) cudaSetDevice(pg->ctx->device);
  if (pg->ctx && pg->ctx->stream) cudaStreamSynchronize(pg->ctx->stream);
  if (pg->h_registered) cudaHostUnregister(pg->h_registered);
  cudaFree(pg->d_arena);
  cudaFree(pg->d_skip_off);
  cudaFree(pg->d_skip);
  cudaFree(pg->d_narrow);
  free_overlap(pg);
  cudaFree(pg->d_descs);
  cudaFree(pg->d_time_page_of);
  cudaFree(pg->d_cg_time_page);
  cudaFree(pg->d_cg_series_rank);
  cudaFree(pg->d_series_sorted);
  cudaFree(pg->d_item_info);
  cudaFree(pg->d_rank_cg_start);
  cudaFree(pg->d_rank_cg);
  cudaFree(pg->d_page_bin);
  cudaFree(pg->d_page_stats);
  cudaFree(pg->d_item_page);
  cudaFree(pg->d_item_cg);
  cudaFree(pg->d_bin_start);
  cudaFree(pg->d_crc_tables);
  cudaFree(pg->d_tomb_keys);
  cudaFree(pg->d_tomb_off);
  cudaFree(pg->d_tomb_ranges);
  cudaFree(pg->d_cg_bounds);
  cudaFree(pg->d_keep_off);
  delete pg;
}

uint64_t tskvgpu_pages_series_count(const tskv_pages *pages) { return pages ? pages->series.size() : 0; }

tskv_status tskvgpu_pages_set_time_bounds(tskv_ctx *ctx, tskv_pages *pg, const tskv_time_range *bounds, uint64_t n) {
  if (!ctx || !pg || !bounds || n != pg->n_cg) return TSKV_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(ctx->mu);
  ctx->set_error("");
  CU_TRY(ctx, cudaSetDevice(ctx->device));
  if (!pg->d_cg_bounds) CU_TRY(ctx, cudaMalloc(reinterpret_cast<void **>(&pg->d_cg_bounds), std::max<size_t>(n, 1) * sizeof(tskv_time_range)));
  CU_TRY(ctx, cudaMemcpy(pg->d_cg_bounds, bounds, n * sizeof(tskv_time_range), cudaMemcpyHostToDevice));
  int64_t lo = INT64_MAX, hi = INT64_MIN;
  for (uint64_t i = 0; i < n; i++)
    if (bounds[i].min_ts <= bounds[i].max_ts) {
      lo = std::min(lo, bounds[i].min_ts);
      hi = std::max(hi, bounds[i].max_ts);
    }
  if (lo <= hi) {
    pg->ts_min = lo;
    pg->ts_max = hi;
  }
  pg->bounds_known = true;
  return TSKV_OK;
}

// PageMeta.statistics of the caller -> the ordered min / max keys the work list prunes with.
tskv_status tskvgpu_pages_set_value_stats(tskv_ctx *ctx, tskv_pages *pg, const tskv_value_stats *stats, uint64_t n_descs) {
  if (!ctx || !pg || !stats || n_descs != pg->n_descs) return TSKV_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(ctx->mu);
  ctx->set_error("");
  CU_TRY(ctx, cudaSetDevice(ctx->device));
  std::vector<int64_t> keys(2 * (size_t)n_descs);
  for (uint64_t i = 0; i < n_descs; i++) {
    const uint8_t pt = pg->h_descs[i].phys_type;
    int64_t kmin = INT64_MIN, kmax = INT64_MAX;  // unknown: nothing can be ruled out
    if ((stats[i].flags & TSKV_STATS_MINMAX) && pt != TSKV_PT_TIME) {
      const bool nan = pt == TSKV_PT_F64 && ((stats[i].min & 0x7fffffffffffffffull) > 0x7ff0000000000000ull ||
                                             (stats[i].max & 0x7fffffffffffffffull) > 0x7ff0000000000000ull);
      if (!nan) {
        kmin = stats_key(stats[i].min, pt);
        kmax = stats_key(stats[i].max, pt);
        if (kmin > kmax) { kmin = INT64_MAX; kmax = INT64_MIN; }  // no value
      }
    }
    keys[2 * i] = kmin;
    keys[2 * i + 1] = kmax;
  }
  CU_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  if (!pg->d_page_stats) CU_TRY(ctx, cudaMalloc(reinterpret_cast<void **>(&pg->d_page_stats), std::max<size_t>(keys.size(), 1) * 8));
  CU_TRY(ctx, cudaMemcpy(pg->d_page_stats, keys.data(), keys.size() * 8, cudaMemcpyHostToDevice));
  return TSKV_OK;
}

// Overlapping chunks: file id of every column group -> merge groups (host_util.h, plan_overlap_groups) + the merge rows'
// timestamps, decoded once.
tskv_status tskvgpu_pages_set_chunk_files(tskv_ctx *ctx, tskv_pages *pg, const uint64_t *cg_file_id, uint64_t n_cg) {
  if (!ctx || !pg || (n_cg && !cg_file_id) || (n_cg && n_cg != pg->n_cg)) return TSKV_ERR_INVALID_ARG;
  {
    std::lock_guard<std::mutex> lock(ctx->mu);
    ctx->set_error("");
    CU_TRY(ctx, cudaSetDevice(ctx->device));
    CU_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    free_overlap(pg);
    pg->chunk_epoch++;
    if (n_cg == 0) return TSKV_OK;
    ensure_time_bounds(ctx, pg);  // ColumnGroup::time_range() of every group (the caller's, or one pass over the time pages)
    if (!pg->d_cg_bounds) {
      ctx->set_error("set_chunk_files: the column groups' time bounds are not available");
      return TSKV_ERR_CUDA;
    }
    pg->h_cg_bounds.resize(pg->n_cg);
    CU_TRY(ctx, cudaMemcpy(pg->h_cg_bounds.data(), pg->d_cg_bounds, (size_t)pg->n_cg * sizeof(tskv_time_range), cudaMemcpyDeviceToHost));
    std::vector<uint32_t> cg_series(pg->n_cg), cg_rows(pg->n_cg);
    for (uint32_t cg = 0; cg < pg->n_cg; cg++) {
      cg_series[cg] = pg->h_descs[pg->h_cg_time_page[cg]].series_id;
      cg_rows[cg] = pg->h_descs[pg->h_cg_time_page[cg]].num_values;
    }
    plan_overlap_groups(pg->n_cg, cg_series.data(), cg_rows.data(), pg->h_cg_bounds.data(), cg_file_id, &pg->overlap);
    const OverlapPlan &op = pg->overlap;
    const size_t n_mcg = op.mcg_cg.size();
    if (n_mcg == 0) return TSKV_OK;  // no two chunks of a series overlap: nothing to merge
    for (uint32_t cg : op.mcg_cg)
      if (pg->h_time_has_nulls[pg->h_cg_time_page[cg]] || dk_is_error(pg->h_descs[pg->h_cg_time_page[cg]].reserved)) {
        ctx->set_error("set_chunk_files: a time page of an overlapping chunk holds NULLs or does not decode", pg->h_cg_time_page[cg]);
        free_overlap(pg);
        return TSKV_ERR_UNSUPPORTED;
      }
    pg->merge_rows = op.mcg_row0.back();
    pg->h_mcg_bm0.assign(n_mcg, 0);
    uint64_t w = 0;
    for (size_t k = 0; k < n_mcg; k++) {
      pg->h_mcg_bm0[k] = w;
      w += ((op.mcg_row0[k + 1] - op.mcg_row0[k] + 63) / 64) * 2;  // 8-byte padded bitmaps, in 32-bit words
    }
    pg->merge_bm_words = w;
    auto up = [&](auto **dptr, const auto &vec) -> cudaError_t {
      cudaError_t e = dev_alloc(dptr, vec.size());
      if (e == cudaSuccess && !vec.empty()) e = cudaMemcpy(*dptr, vec.data(), vec.size() * sizeof(vec[0]), cudaMemcpyHostToDevice);
      return e;
    };
    cudaError_t e = up(&pg->d_cg_merge, op.cg_merge);
    if (e == cudaSuccess) e = up(&pg->d_mcg_row0, op.mcg_row0);
    if (e == cudaSuccess) e = up(&pg->d_mcg_bm0, pg->h_mcg_bm0);
    if (e == cudaSuccess) e = up(&pg->d_mcg_cg, op.mcg_cg);
    if (e == cudaSuccess) e = up(&pg->d_mcg_stream, op.mcg_stream);
    if (e == cudaSuccess) e = up(&pg->d_stream_group, op.stream_group);
    if (e == cudaSuccess) e = up(&pg->d_stream_first_mcg, op.stream_first_mcg);
    if (e == cudaSuccess) e = up(&pg->d_group_first_stream, op.group_first_stream);
    if (e == cudaSuccess) e = dev_alloc(&pg->d_merge_ts, (size_t)pg->merge_rows);
    // the merge rows' timestamps: the time pages of the merge column groups, decoded in merge-row order
    std::vector<uint32_t> tpages(n_mcg);
    std::vector<uint64_t> row_off(n_mcg), bm_off(n_mcg);
    for (size_t k = 0; k < n_mcg; k++) {
      tpages[k] = pg->h_cg_time_page[op.mcg_cg[k]];
      row_off[k] = op.mcg_row0[k];
      bm_off[k] = pg->h_mcg_bm0[k] * 4;
    }
    uint32_t *d_list = nullptr;
    uint64_t *d_ro = nullptr, *d_bo = nullptr;
    uint8_t *d_bm = nullptr;
    int32_t *d_st = nullptr;
    if (e == cudaSuccess) e = up(&d_list, tpages);
    if (e == cudaSuccess) e = up(&d_ro, row_off);
    if (e == cudaSuccess) e = up(&d_bo, bm_off);
    if (e == cudaSuccess) e = dev_alloc(&d_bm, (size_t)pg->merge_bm_words * 4);
    if (e == cudaSuccess) e = dev_alloc(&d_st, 8);  // status | err page (2 x 8 bytes) | points
    tskv_status ret = TSKV_OK;
    if (e == cudaSuccess) e = cudaMemsetAsync(d_st, 0, 32, ctx->stream);
    if (e == cudaSuccess) {
      unsigned long long *aux = reinterpret_cast<unsigned long long *>(d_st);
      const uint32_t blocks = (uint32_t)((n_mcg * 32 + DECODE_THREADS - 1) / DECODE_THREADS);
      k_decode_warp<<<blocks, DECODE_THREADS, 0, ctx->stream>>>(pg->h_mapped ? pg->h_mapped : pg->d_arena, pg->d_descs, 0, d_list, (uint32_t)n_mcg,
                                                               d_ro, d_bo, reinterpret_cast<uint64_t *>(pg->d_merge_ts), d_bm, d_st, aux + 1, aux + 2);
      e = cudaGetLastError();
      if (e == cudaSuccess) ret = fetch_status(ctx, d_st, aux + 1);
    }
    cudaFree(d_list); cudaFree(d_ro); cudaFree(d_bo); cudaFree(d_bm); cudaFree(d_st);
    if (e != cudaSuccess || ret != TSKV_OK) {
      if (e != cudaSuccess) ctx->set_error(std::string("set_chunk_files: ") + cudaGetErrorString(e));
      free_overlap(pg);
      return e == cudaErrorMemoryAllocation ? TSKV_ERR_OOM : (e != cudaSuccess ? TSKV_ERR_CUDA : ret);
    }
  }
  return TSKV_OK;
}

// TsmTombstone cache -> device tables: the all-series ranges first, then one CSR row per (series, column) key.
tskv_status tskvgpu_pages_set_tombstones(tskv_ctx *ctx, tskv_pages *pg, const tskv_tombstone *tombs, uint64_t n_tombs) {
  if (!ctx || !pg || (n_tombs && !tombs) || n_tombs > 0x7fffffffull) return TSKV_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(ctx->mu);
  ctx->set_error("");
  CU_TRY(ctx, cudaSetDevice(ctx->device));
  std::vector<tskv_time_range> ranges;
  std::vector<std::pair<uint64_t, tskv_time_range>> keyed;
  for (uint64_t i = 0; i < n_tombs; i++) {
    const tskv_tombstone &tb = tombs[i];
    if (tb.series_id == TSKV_TOMB_ALL && tb.column_id != TSKV_TOMB_ALL) {
      ctx->set_error("tombstone: series_id = TSKV_TOMB_ALL needs column_id = TSKV_TOMB_ALL", -1);
      return TSKV_ERR_INVALID_ARG;
    }
    if (tb.min_ts > tb.max_ts) continue;  // empty range
    if (tb.series_id == TSKV_TOMB_ALL) ranges.push_back({tb.min_ts, tb.max_ts});
    else keyed.push_back({((uint64_t)tb.series_id << 32) | tb.column_id, {tb.min_ts, tb.max_ts}});
  }
  std::stable_sort(keyed.begin(), keyed.end(), [](const auto &a, const auto &b) { return a.first < b.first; });
  const uint32_t n_global = (uint32_t)ranges.size();
  std::vector<uint64_t> keys;
  std::vector<uint32_t> off;
  for (const auto &kr : keyed) {
    if (keys.empty() || keys.back() != kr.first) {
      keys.push_back(kr.first);
      off.push_back((uint32_t)ranges.size());
    }
    ranges.push_back(kr.second);
  }
  off.push_back((uint32_t)ranges.size());
  CU_TRY(ctx, cudaStreamSynchronize(ctx->stream));  // no scan of this page set may be in flight
  cudaFree(pg->d_tomb_keys);
  cudaFree(pg->d_tomb_off);
  cudaFree(pg->d_tomb_ranges);
  pg->d_tomb_keys = nullptr;
  pg->d_tomb_off = nullptr;
  pg->d_tomb_ranges = nullptr;
  pg->n_tomb_keys = (uint32_t)keys.size();
  pg->n_tomb_global = n_global;
  pg->n_tomb_ranges = (uint32_t)ranges.size();
  pg->tomb_epoch++;
  if (!ranges.empty()) {
    CU_TRY(ctx, cudaMalloc(&pg->d_tomb_ranges, ranges.size() * sizeof(tskv_time_range)));
    CU_TRY(ctx, cudaMemcpy(pg->d_tomb_ranges, ranges.data(), ranges.size() * sizeof(tskv_time_range), cudaMemcpyHostToDevice));
    CU_TRY(ctx, cudaMalloc(&pg->d_tomb_keys, std::max<size_t>(keys.size(), 1) * 8));
    if (!keys.empty()) CU_TRY(ctx, cudaMemcpy(pg->d_tomb_keys, keys.data(), keys.size() * 8, cudaMemcpyHostToDevice));
    CU_TRY(ctx, cudaMalloc(&pg->d_tomb_off, off.size() * 4));
    CU_TRY(ctx, cudaMemcpy(pg->d_tomb_off, off.data(), off.size() * 4, cudaMemcpyHostToDevice));
  }
  return TSKV_OK;
}

// ------------------------------------------------------------------------------------------------
tskv_status tskvgpu_decode_pages(tskv_ctx *ctx, const tskv_pages *pages, uint64_t first_page,
                                 uint64_t n_pages, uint64_t *out_values, uint8_t *out_validity) {
  if (!ctx || !pages || n_pages > pages->n_descs || first_page > pages->n_descs - n_pages || (n_pages && (!out_values || !out_validity)))
    return TSKV_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(ctx->mu);
  ctx->set_error("");
  if (n_pages == 0) return TSKV_OK;
  cudaSetDevice(ctx->device);
  std::vector<uint64_t> row_off(n_pages), bm_off(n_pages);
  uint64_t rows = 0, bm = 0;
  for (uint64_t i = 0; i < n_pages; i++) {
    row_off[i] = rows;
    bm_off[i] = bm;
    rows += pages->h_descs[first_page + i].num_values;
    bm += ((uint64_t)pages->h_descs[first_page + i].num_values + 63) / 64 * 8;
  }
  uint64_t *d_row_off = nullptr, *d_bm_off = nullptr, *d_vals = nullptr;
  uint8_t *d_valid = nullptr;
  int32_t *d_status = nullptr;
  unsigned long long *d_aux = nullptr;  // [0] err_page, [1] points
  tskv_status ret = TSKV_OK;
  auto cleanup = [&]() {
    cudaFree(d_row_off);
    cudaFree(d_bm_off);
    cudaFree(d_vals);
    cudaFree(d_valid);
    cudaFree(d_status);
    cudaFree(d_aux);
  };
  cudaError_t e = dev_alloc(&d_row_off, n_pages);
  if (e == cudaSuccess) e = dev_alloc(&d_bm_off, n_pages);
  if (e == cudaSuccess) e = dev_alloc(&d_vals, rows);
  if (e == cudaSuccess) e = dev_alloc(&d_valid, bm);
  if (e == cudaSuccess) e = dev_alloc(&d_status, 1);
  if (e == cudaSuccess) e = dev_alloc(&d_aux, 2);
  if (e == cudaSuccess) e = cudaMemcpyAsync(d_row_off, row_off.data(), n_pages * 8, cudaMemcpyHostToDevice, ctx->stream);
  if (e == cudaSuccess) e = cudaMemcpyAsync(d_bm_off, bm_off.data(), n_pages * 8, cudaMemcpyHostToDevice, ctx->stream);
  if (e == cudaSuccess) e = cudaMemsetAsync(d_status, 0, 4, ctx->stream);
  if (e == cudaSuccess) e = cudaMemsetAsync(d_aux, 0, 16, ctx->stream);
  if (e == cudaSuccess) e = cudaMemsetAsync(d_vals, 0, std::max<uint64_t>(rows, 1) * 8, ctx->stream);
  if (e == cudaSuccess) {
    cudaEventRecord(ctx->ev0, ctx->stream);
    uint32_t blocks = (uint32_t)((n_pages * 32 + DECODE_THREADS - 1) / DECODE_THREADS);  // one warp per page
    // host-resident page sets: d_arena is only the scans' gather target, the pages are read through the mapped host range
    k_decode_warp<<<blocks, DECODE_THREADS, 0, ctx->stream>>>(pages->h_mapped ? pages->h_mapped : pages->d_arena, pages->d_descs, first_page, nullptr, (uint32_t)n_pages,
                                                        d_row_off, d_bm_off, d_vals, d_valid, d_status, d_aux, d_aux + 1);
    cudaEventRecord(ctx->ev1, ctx->stream);
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaMemcpyAsync(out_values, d_vals, rows * 8, cudaMemcpyDeviceToHost, ctx->stream);
  if (e == cudaSuccess) e = cudaMemcpyAsync(out_validity, d_valid, bm, cudaMemcpyDeviceToHost, ctx->stream);
  unsigned long long points = 0;
  if (e == cudaSuccess) e = cudaMemcpyAsync(&points, d_aux + 1, 8, cudaMemcpyDeviceToHost, ctx->stream);
  if (e == cudaSuccess) {
    ret = fetch_status(ctx, d_status, d_aux);
  } else {
    ctx->set_error(std::string("decode: ") + cudaGetErrorString(e));
    ret = e == cudaErrorMemoryAllocation ? TSKV_ERR_OOM : TSKV_ERR_CUDA;
  }
  if (ret == TSKV_OK) {
    float ms = 0;
    cudaEventElapsedTime(&ms, ctx->ev0, ctx->ev1);
    ctx->counters.elapsed_scan_ms = ms;
    ctx->counters.points_decoded = points;
    ctx->counters.kernel_launches = 1;
    ctx->counters.page_read_count = n_pages;
  }
  cleanup();
  return ret;
}

// ------------------------------------------------------------------------------------------------
tskv_status tskvgpu_query_output_layout(const tskv_pages *pages, const tskv_query *q,
                                        tskv_output_layout *out) {
  return compute_layout(pages, q, TagGroups{}, out);
}

tskv_status tskvgpu_query_output_layout_grouped(const tskv_pages *pages, const tskv_query *q, const uint32_t *group_ids,
                                                uint32_t n_groups, tskv_output_layout *out) {
  return compute_layout(pages, q, TagGroups{true, group_ids, n_groups}, out);
}

// Sliding windows of `q` (window q->width, slide < q->width) by panes: the refusals of tskvgpu_scan_prepare_sliding
// (DESIGN.md section 7) and the pane grid. Called under ctx->mu.
static tskv_status check_sliding(tskv_ctx *ctx, const tskv_pages *pages, const tskv_query *q, int64_t slide, uint32_t *out_k) {
  for (uint32_t c = 0; c < q->n_columns; c++)
    if (q->columns[c].agg_mask & (TSKV_AGG_FIRST | TSKV_AGG_LAST)) {
      ctx->set_error("sliding windows: FIRST / LAST drop a (page, window) run on a NULL at its first / last row, which "
                     "pane partials cannot rebuild");
      return TSKV_ERR_UNSUPPORTED;
    }
  if (slide > q->width) {
    ctx->set_error("sliding windows: a slide wider than the window (rows between windows) is not pushed down");
    return TSKV_ERR_UNSUPPORTED;
  }
  if (q->width >= (int64_t)1 << 61) {
    ctx->set_error("sliding windows: window of 2^61 or more");
    return TSKV_ERR_UNSUPPORTED;
  }
  const uint64_t k = ((uint64_t)q->width - 1) / (uint64_t)slide + 1;  // windows per row, ceil(window / slide)
  if (k > 100) {
    ctx->set_error("sliding windows: more than 100 windows per row (Too many overlapping windows)");
    return TSKV_ERR_INVALID_ARG;
  }
  if (q->n_buckets < k) {
    ctx->set_error("sliding windows: n_buckets must be at least ceil(window / slide)");
    return TSKV_ERR_INVALID_ARG;
  }
  if ((unsigned __int128)q->n_buckets * (uint64_t)slide > (unsigned __int128)1 << 63) {
    ctx->set_error("sliding windows: the window grid spans more than 2^63");
    return TSKV_ERR_INVALID_ARG;
  }
  // With window % slide != 0 the reference keeps a row's copies by the test window-0 start <= t < end, which passes for
  // every row whose dividend t - start_time % window + slide is >= 0 and whose window end does not wrap, and fails for
  // other rows unless the remainder is 0: refuse unless every row the query can select is of the first kind.
  if (q->width % slide != 0 && pages->n_cg) {
    ensure_time_bounds(ctx, pages);
    int64_t lo = pages->ts_min, hi = pages->ts_max;
    if (q->n_time_ranges > 0) {
      int64_t qlo = q->time_ranges[0].min_ts, qhi = q->time_ranges[0].max_ts;
      for (uint32_t r = 1; r < q->n_time_ranges; r++) {
        qlo = std::min(qlo, q->time_ranges[r].min_ts);
        qhi = std::max(qhi, q->time_ranges[r].max_ts);
      }
      lo = std::max(lo, qlo);
      hi = std::min(hi, qhi);
    }
    const __int128 om = q->origin % q->width;
    if (lo <= hi && ((__int128)lo - om + slide < 0 || (__int128)hi - om + slide > (__int128)INT64_MAX ||
                     (__int128)hi + q->width > (__int128)INT64_MAX)) {
      ctx->set_error("sliding windows: window % slide != 0 and rows in the truncating-% or wrapping range of the window "
                     "expression");
      return TSKV_ERR_UNSUPPORTED;
    }
  }
  *out_k = (uint32_t)k;
  return TSKV_OK;
}

// tskvgpu_scan_prepare; slide > 0: tskvgpu_scan_prepare_sliding with slide < width; tg.on: GROUP BY tags.
static tskv_status prepare_scan(tskv_ctx *ctx, const tskv_pages *pages, const tskv_query *q, int64_t slide,
                                const TagGroups &tg, tskv_scan **out_scan) {
  if (!ctx || !pages || !q || !out_scan) return TSKV_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(ctx->mu);
  ctx->set_error("");
  *out_scan = nullptr;
  if (const char *why = tag_groups_refusal(pages, q, tg)) {
    ctx->set_error(why);
    return TSKV_ERR_INVALID_ARG;
  }
  tskv_output_layout L;
  tskv_status st = compute_layout(pages, q, tg, &L);
  if (st != TSKV_OK) {
    ctx->set_error("invalid query (buckets / columns)");
    return st;
  }
  if (q->n_columns > 126 || q->n_time_ranges > MAX_RANGES || (q->n_time_ranges && !q->time_ranges) ||
      (q->series_ids == nullptr && q->n_series != 0 && false)) {
    ctx->set_error("invalid query: at most 126 columns and 8 time ranges");
    return TSKV_ERR_INVALID_ARG;
  }
  if (q->n_predicates > TSKV_MAX_PREDICATES || (q->n_predicates && !q->predicates)) {
    ctx->set_error("invalid query: at most 8 field predicates");
    return TSKV_ERR_INVALID_ARG;
  }
  for (uint32_t k = 0; k < q->n_predicates; k++)
    if (q->predicates[k].phys_type < TSKV_PT_I64 || q->predicates[k].phys_type > TSKV_PT_F64 || q->predicates[k].op > TSKV_CMP_GE) {
      ctx->set_error("invalid field predicate (type or operator)");
      return TSKV_ERR_INVALID_ARG;
    }
  for (uint32_t c = 0; c < q->n_columns; c++) {
    const tskv_agg_column &qc = q->columns[c];
    if (qc.phys_type < TSKV_PT_I64 || qc.phys_type > TSKV_PT_BOOL || (qc.agg_mask & ~TSKV_AGG_ALL) || qc.agg_mask == 0) {
      ctx->set_error("invalid query column (type or aggregate mask)");
      return TSKV_ERR_INVALID_ARG;
    }
    if (qc.phys_type == TSKV_PT_BOOL && (qc.agg_mask & (TSKV_AGG_SUM | TSKV_AGG_MEAN))) {
      ctx->set_error("sum / mean of a boolean column");
      return TSKV_ERR_INVALID_ARG;
    }
    for (uint32_t c2 = 0; c2 < c; c2++)
      if (q->columns[c2].column_id == qc.column_id) {
        ctx->set_error("duplicate query column id");
        return TSKV_ERR_INVALID_ARG;
      }
  }
  if (q->series_ids)
    for (uint32_t i = 1; i < q->n_series; i++)
      if (q->series_ids[i] <= q->series_ids[i - 1]) {
        ctx->set_error("series_ids must be sorted ascending and unique");
        return TSKV_ERR_INVALID_ARG;
      }
  if ((q->reserved & TSKV_QUERY_MULTI_RANK) && !q->series_ids) {
    bool needs_slots = q->group_by_series != 0 || tg.on;
    for (uint32_t c = 0; c < q->n_columns; c++) needs_slots |= (q->columns[c].agg_mask & (TSKV_AGG_FIRST | TSKV_AGG_LAST)) != 0;
    if (needs_slots) {
      ctx->set_error("multi-rank scan: GROUP BY series / tags and first/last need the global series_ids list (slots are positions in it)");
      return TSKV_ERR_INVALID_ARG;
    }
  }
  uint32_t win_k = 1;
  if (slide) {
    st = check_sliding(ctx, pages, q, slide, &win_k);
    if (st != TSKV_OK) return st;
  }
  cudaSetDevice(ctx->device);
  tskv_scan *s = new tskv_scan();
  s->pages = pages;
  s->layout = L;
  s->n_cols = q->n_columns;
  s->n_out = (uint32_t)L.n_out;
  const uint64_t n_cells = L.n_cells;
  // the fused kernels' bucket grid: the query's, or for a sliding scan the panes of width `slide`, from the start of the
  // last pane of window 0 to the start of the last window
  s->win_k = win_k;
  s->n_windows = q->n_buckets;
  s->n_panes = q->n_buckets - win_k + 1;
  const uint64_t kern_cells = L.n_groups * s->n_panes;

  // ---- first/last key budget ---------------------------------------------------------------------
  bool any_sel = false;
  for (uint32_t c = 0; c < q->n_columns; c++) any_sel |= (q->columns[c].agg_mask & (TSKV_AGG_FIRST | TSKV_AGG_LAST)) != 0;
  s->has_sel = any_sel;
  uint64_t n_slots = q->series_ids ? q->n_series : pages->series.size();
  uint32_t slot_bits = (q->group_by_series || n_slots <= 1) ? 0 : bits_for(n_slots - 1);
  int64_t rel_base = 0;
  if (any_sel && slot_bits > 0) {
    unsigned rel_bits = 64;
    if (q->width > 0) {
      if (q->width < (int64_t)1 << 61) rel_bits = bits_for(2 * (uint64_t)q->width);
    } else {
      // unbucketed: rel = t - (lower bound of every in-range timestamp). A single-rank scan tightens unbounded / loose
      // query ranges with the arena's own time bounds; a scan whose partials are merged with other ranks'
      // (TSKV_QUERY_MULTI_RANK) must build keys every rank agrees on, i.e. from the query alone.
      const bool multi_rank = (q->reserved & TSKV_QUERY_MULTI_RANK) != 0;
      int64_t lo = INT64_MIN, hi = INT64_MAX;
      if (!multi_rank) {
        ensure_time_bounds(ctx, pages);
        lo = pages->ts_min;
        hi = pages->ts_max;
      }
      if (q->n_time_ranges > 0) {
        int64_t qlo = q->time_ranges[0].min_ts, qhi = q->time_ranges[0].max_ts;
        for (uint32_t k = 1; k < q->n_time_ranges; k++) {
          qlo = std::min(qlo, q->time_ranges[k].min_ts);
          qhi = std::max(qhi, q->time_ranges[k].max_ts);
        }
        lo = std::max(lo, qlo);
        hi = std::min(hi, qhi);
      }
      if (hi < lo) {
        rel_bits = 0;  // nothing can be in range
      } else {
        uint64_t span = (uint64_t)hi - (uint64_t)lo;
        rel_bits = bits_for(span);
        rel_base = lo;
      }
    }
    if (rel_bits + slot_bits > 62) {
      ctx->set_error("first/last across series: (bucket width or time span) x series count does not fit the 62-bit tie-break key");
      delete s;
      return TSKV_ERR_UNSUPPORTED;
    }
  }

  // ---- state layout ------------------------------------------------------------------------------
  // a sliding scan: what the fused kernels write (panes) and what the rest of the pass sees (windows)
  const StatePlan win = plan_state(q, n_cells);
  const StatePlan pane = slide ? plan_state(q, kern_cells) : StatePlan{};
  s->sl = win.sl;
  s->kern_sl = slide ? pane.sl : win.sl;
  std::vector<ColState> cols = slide ? pane.cols : win.cols;
  const std::vector<MeanExport> &means = win.means;
  const std::vector<uint64_t> &msum_off = win.msum_off;
  const StateLayout &sl = s->sl;
  std::vector<CombineOp> combine;
  if (slide) {
    for (uint32_t c = 0; c < q->n_columns; c++) {
      const ColState &p = pane.cols[c], &w = win.cols[c];
      const uint8_t m = q->columns[c].agg_mask;
      combine.push_back(CombineOp{p.count_off, w.count_off, 0, 0, COMBINE_ADD, 0});
      if (m & (TSKV_AGG_SUM | TSKV_AGG_MEAN)) {
        if (q->columns[c].phys_type == TSKV_PT_F64) combine.push_back(CombineOp{p.sum_off, w.sum_off, 0, 0, COMBINE_F64_SUM, 0});
        else combine.push_back(CombineOp{p.sum_off, w.sum_off, p.sumhi_off, w.sumhi_off, COMBINE_INT_SUM, (m & TSKV_AGG_MEAN) ? 1u : 0u});
      }
      if (m & TSKV_AGG_MIN) combine.push_back(CombineOp{p.min_off, w.min_off, 0, 0, COMBINE_MIN, 0});
      if (m & TSKV_AGG_MAX) combine.push_back(CombineOp{p.max_off, w.max_off, 0, 0, COMBINE_MAX, 0});
    }
  }

  // output column table
  std::vector<OutCol> outs;
  {
    uint64_t fk = sl.first_keys_off, lk = sl.last_keys_off, fv = sl.selval_off, lv = sl.selval_off + sl.first_cells;
    for (uint32_t c = 0; c < q->n_columns; c++) {
      const tskv_agg_column &qc = q->columns[c];
      for (unsigned bit = 0; bit < 7; bit++) {
        unsigned agg = 1u << bit;
        if (!(qc.agg_mask & agg)) continue;
        OutCol oc{};
        oc.count_off = win.cols[c].count_off;
        oc.agg = (uint8_t)agg;
        oc.phys_type = qc.phys_type;
        switch (agg) {
          case TSKV_AGG_SUM: oc.src_off = win.cols[c].sum_off; break;
          case TSKV_AGG_MEAN: oc.src_off = msum_off[c] ? msum_off[c] : win.cols[c].sum_off; break;
          case TSKV_AGG_MIN: oc.src_off = win.cols[c].min_off; break;
          case TSKV_AGG_MAX: oc.src_off = win.cols[c].max_off; break;
          case TSKV_AGG_FIRST: oc.src_off = fk; oc.val_off = fv; break;
          case TSKV_AGG_LAST: oc.src_off = lk; oc.val_off = lv; break;
          default: break;
        }
        outs.push_back(oc);
      }
      if (qc.agg_mask & TSKV_AGG_FIRST) { fk += n_cells; fv += n_cells; }
      if (qc.agg_mask & TSKV_AGG_LAST) { lk += n_cells; lv += n_cells; }
    }
  }

  // ---- device allocations (stream-ordered) + query arguments H2D --------------------------------------
  const uint32_t n_items = pages->n_items;
  s->ctx = ctx;
  cudaEventCreate(&s->ev0);
  cudaEventCreate(&s->ev1);
  for (int b = 0; b <= N_BINS; b++) cudaEventCreate(&s->ev_bin[b]);
  for (int b = 0; b < N_BINS; b++) {
    cudaEventCreate(&s->ev_bin_start[b]);
    cudaEventCreate(&s->ev_bin_done[b]);
    cudaEventCreateWithFlags(&s->ev_gather[b], cudaEventDisableTiming);
  }
  s->n_series_sel = q->series_ids ? q->n_series : 0;
  s->n_blocks = (n_items + 1023) / 1024;
  cudaError_t e = cudaSuccess;
  uint64_t h2d = 0;
  if (q->series_ids) {
    e = stream_alloc(ctx, &s->d_series, q->n_series);
    if (e == cudaSuccess && q->n_series)
      e = cudaMemcpyAsync(s->d_series, q->series_ids, (size_t)q->n_series * 4, cudaMemcpyHostToDevice, ctx->stream);
    h2d += (uint64_t)q->n_series * 4;
  }
  if (tg.on) {  // GROUP BY tags: the group map, and the slots in group order for the work-list walk
    const uint64_t n_slots = selected_slots(pages, q);
    std::vector<uint32_t> walk;
    if (!std::is_sorted(tg.ids, tg.ids + n_slots)) {  // (already in group order: the walk stays the selection order)
      walk.resize(n_slots);
      if (tg.n <= n_slots) {  // stable counting sort
        std::vector<uint32_t> next(tg.n + 1, 0);
        for (uint64_t i = 0; i < n_slots; i++) next[tg.ids[i] + 1]++;
        for (uint32_t g = 0; g < tg.n; g++) next[g + 1] += next[g];
        for (uint64_t i = 0; i < n_slots; i++) walk[next[tg.ids[i]]++] = (uint32_t)i;
      } else {
        std::iota(walk.begin(), walk.end(), 0u);
        std::stable_sort(walk.begin(), walk.end(), [&](uint32_t a, uint32_t b) { return tg.ids[a] < tg.ids[b]; });
      }
    }
    if (e == cudaSuccess) e = stream_alloc(ctx, &s->d_slot_group, n_slots);
    if (e == cudaSuccess && n_slots)
      e = cudaMemcpyAsync(s->d_slot_group, tg.ids, (size_t)n_slots * 4, cudaMemcpyHostToDevice, ctx->stream);
    if (e == cudaSuccess && !walk.empty()) e = stream_alloc(ctx, &s->d_walk, n_slots);
    if (e == cudaSuccess && !walk.empty())
      e = cudaMemcpyAsync(s->d_walk, walk.data(), (size_t)n_slots * 4, cudaMemcpyHostToDevice, ctx->stream);
    h2d += (n_slots + walk.size()) * 4;
  }
  if (e == cudaSuccess && q->series_ids) e = stream_alloc(ctx, &s->d_rank_slot, pages->series.size());
  if (e == cudaSuccess) e = stream_alloc(ctx, &s->d_bucket, (size_t)2 * N_BINS * q->n_columns * WL_SUB + 1);
  {
    // One thread walks ALL column groups of a selected series: right for many series with a few groups each (TSBS
    // shapes), serial for a handful of series with thousands of groups (one host over a year) - those take the pass
    // over every field page instead, which is parallel in the pages. TSKV_WORKLIST=items / series forces one.
    const char *wl = getenv("TSKV_WORKLIST");
    s->worklist_by_items = wl ? wl[0] == 'i' : (uint64_t)pages->n_cg > 32ull * std::max<uint64_t>(1, pages->series.size());
  }
  if (e == cudaSuccess) e = stream_alloc(ctx, &s->d_cg_slot, pages->n_cg);
  if (e == cudaSuccess) e = stream_alloc(ctx, &s->d_item_flag, n_items);
  if (e == cudaSuccess) e = stream_alloc(ctx, &s->d_block_count, s->n_blocks);
  if (e == cudaSuccess) e = stream_alloc(ctx, &s->d_work_page, n_items);
  if (e == cudaSuccess) e = stream_alloc(ctx, &s->d_work_slot, n_items);
  if (e == cudaSuccess) e = stream_alloc(ctx, &s->d_work_qcol, n_items);
  if (e == cudaSuccess) e = stream_alloc(ctx, &s->d_bin_cstart, N_BINS + 2);
  if (e == cudaSuccess) e = stream_alloc(ctx, &s->d_cols, cols.size());
  if (e == cudaSuccess) e = stream_alloc(ctx, &s->d_outs, outs.size());
  s->n_means = (uint32_t)means.size();
  if (e == cudaSuccess) e = stream_alloc(ctx, &s->d_means, means.size());
  if (e == cudaSuccess && !means.empty())
    e = cudaMemcpyAsync(s->d_means, means.data(), means.size() * sizeof(MeanExport), cudaMemcpyHostToDevice, ctx->stream);
  if (e == cudaSuccess) e = stream_alloc(ctx, &s->d_state, sl.total);
  if (e == cudaSuccess && slide) e = stream_alloc(ctx, &s->d_pane_state, s->kern_sl.total);
  s->n_combine = (uint32_t)combine.size();
  if (e == cudaSuccess && slide) e = stream_alloc(ctx, &s->d_combine, combine.size());
  if (e == cudaSuccess && slide)
    e = cudaMemcpyAsync(s->d_combine, combine.data(), combine.size() * sizeof(CombineOp), cudaMemcpyHostToDevice, ctx->stream);
  s->preds.n = q->n_predicates;
  for (uint32_t k = 0; k < q->n_predicates; k++) s->preds.p[k] = q->predicates[k];
  if (q->n_predicates) ensure_page_stats(ctx, pages);  // value-statistics pruning (filter_column_groups, reader/chunk.rs:12-50)
  if (e == cudaSuccess && q->n_predicates) e = stream_alloc(ctx, &s->d_row_keep, (size_t)pages->keep_words);
  // aux block (8-byte units): [0..7] task counters (N_BINS x u32) | 8 status | 9 err_page | 10,11 stats
  //                           | 12 pages 13 bytes 14..22 per-bin bytes
  if (e == cudaSuccess) e = stream_alloc(ctx, reinterpret_cast<unsigned long long **>(&s->d_task_counter), 32);
  if (e == cudaSuccess) e = stream_alloc(ctx, &s->d_values, L.n_out * L.n_cells);
  if (e == cudaSuccess) e = stream_alloc(ctx, &s->d_validity, L.validity_bytes + 8);
  if (e == cudaSuccess) e = cudaMemcpyAsync(s->d_outs, outs.data(), outs.size() * sizeof(OutCol), cudaMemcpyHostToDevice, ctx->stream);
  h2d += cols.size() * sizeof(ColState) + outs.size() * sizeof(OutCol) + means.size() * sizeof(MeanExport) + sizeof(ScanParams) +
         combine.size() * sizeof(CombineOp);
  if (e != cudaSuccess) {
    ctx->set_error(std::string("scan_prepare: ") + cudaGetErrorString(e));
    free_scan(s);
    return e == cudaErrorMemoryAllocation ? TSKV_ERR_OOM : TSKV_ERR_CUDA;
  }
  unsigned long long *aux = reinterpret_cast<unsigned long long *>(s->d_task_counter);
  s->d_status = reinterpret_cast<int32_t *>(aux + 8);
  s->d_err_page = aux + 9;
  s->d_stats = aux + 10;
  s->d_counters = aux + 12;
  s->d_crc_status = reinterpret_cast<int32_t *>(aux + 28);
  s->d_crc_err_page = aux + 29;
  cudaEventCreateWithFlags(&s->ev_crc, cudaEventDisableTiming);
  cudaEventCreateWithFlags(&s->ev_ccrc, cudaEventDisableTiming);

  // ---- kernel parameters ------------------------------------------------------------------------------
  ScanParams &P = s->params;
  P.arena = pages->d_arena;
  P.descs = pages->d_descs;
  P.time_page_of = pages->d_time_page_of;
  P.work_page = s->d_work_page;
  P.work_slot = s->d_work_slot;
  P.work_qcol = s->d_work_qcol;
  P.bin_cstart = s->d_bin_cstart;
  P.cols = s->d_cols;
  P.state = slide ? s->d_pane_state : s->d_state;
  P.task_counter = s->d_task_counter;
  P.status = s->d_status;
  P.err_page = s->d_err_page;
  P.stats = s->d_stats;
  P.n_ranges = q->n_time_ranges;
  for (uint32_t k = 0; k < q->n_time_ranges; k++) P.ranges[k] = q->time_ranges[k];
  if (q->n_time_ranges) {  // statistics pruning needs the groups' time bounds (one pass over the time pages, once per page set)
    ensure_time_bounds(ctx, pages);
    s->prune.n = q->n_time_ranges;
    for (uint32_t k = 0; k < q->n_time_ranges; k++) s->prune.r[k] = q->time_ranges[k];
  }
  P.width = slide ? slide : q->width;
  P.origin_mod = q->width > 0 ? q->origin % q->width : 0;  // (a sliding scan: start_time % window, as the reference)
  if (P.width > 0) {
    const __int128 cap = (__int128)INT64_MAX - ((__int128)P.width - P.origin_mod);
    const __int128 wlo = (__int128)INT64_MIN + ((__int128)P.origin_mod - P.width);
    P.floor_cap = cap > (__int128)INT64_MAX ? INT64_MAX : (int64_t)cap;
    P.wrap_lo = wlo < (__int128)INT64_MIN ? INT64_MIN : (int64_t)wlo;
  }
  P.first_bucket_start = (int64_t)((uint64_t)q->first_bucket_start + (uint64_t)(win_k - 1) * (uint64_t)P.width);
  P.n_buckets = s->n_panes;
  P.group_by_series = q->group_by_series;
  P.n_cells = kern_cells;
  P.slot_group = s->d_slot_group;
  P.slot_bits = slot_bits;
  P.slot_max = slot_bits ? (uint32_t)((1ull << slot_bits) - 1) : 0;
  P.rel_base = rel_base;
  // per-CTA shared-memory partial table (GROUP BY bucket / tags): count | sum | hi | min | max per column
  {
    uint32_t words = 0;
    for (uint32_t c = 0; c < q->n_columns; c++) {
      const uint8_t m = q->columns[c].agg_mask;
      const bool is_int = q->columns[c].phys_type != TSKV_PT_F64;
      cols[c].s_count = words; words += (uint32_t)kern_cells;
      if (m & (TSKV_AGG_SUM | TSKV_AGG_MEAN)) { cols[c].s_sum = words; words += (uint32_t)kern_cells; }
      if ((m & TSKV_AGG_MEAN) && is_int) { cols[c].s_hi = words; words += (uint32_t)kern_cells; }
      if (m & TSKV_AGG_MIN) { cols[c].s_min = words; words += (uint32_t)kern_cells; }
      if (m & TSKV_AGG_MAX) { cols[c].s_max = words; words += (uint32_t)kern_cells; }
      if (kern_cells > (1u << 20)) { words = UINT32_MAX / 2; break; }
    }
    // table limit 32 KB: larger tables cost more in occupancy than the contention they remove (H100, C3: 10 columns x
    // 168 buckets, 53 KB table: 7.8 ms vs 5.4 ms with global atomics); TSKV_SMEM_TABLE_KB overrides
    const char *lim_env = getenv("TSKV_SMEM_TABLE_KB");
    const uint64_t limit = (lim_env ? (uint64_t)atoi(lim_env) : 32) * 1024;
    P.use_smem = (!q->group_by_series && (uint64_t)words * 8 <= limit) ? 1u : 0u;
    P.smem_words = P.use_smem ? words : 0;
    P.n_cols = q->n_columns;
    P.row_keep = s->d_row_keep;
    P.keep_off = pages->d_keep_off;
    P.skip_off = pages->d_skip_off;
    P.page_narrow = pages->d_narrow;
    P.skip = pages->d_skip;
    for (int b = 0; b < N_BINS; b++) { P.bin_parts[b] = 1; P.bin_part_rows[b] = 0; }
    P.has_tomb = pages->n_tomb_ranges ? 1u : 0u;
    P.tomb_keys = pages->d_tomb_keys;
    P.tomb_off = pages->d_tomb_off;
    P.tomb_ranges = pages->d_tomb_ranges;
    P.n_tomb_keys = pages->n_tomb_keys;
    P.n_tomb_global = pages->n_tomb_global;
    s->tomb_epoch = pages->tomb_epoch;
  }
  if (cudaMemcpyAsync(s->d_cols, cols.data(), cols.size() * sizeof(ColState), cudaMemcpyHostToDevice, ctx->stream) != cudaSuccess) {
    ctx->set_error("scan_prepare: column table upload failed");
    free_scan(s);
    return TSKV_ERR_CUDA;
  }

  {
    const double sel_frac = plan_selected_fraction(pages->series.data(), pages->series.size(), q->series_ids, q->n_series);
    // Grid sizes. Every kernel is persistent (warps pull tasks from their bin's counter). If the resident
    // capacity allows, each bin gets one warp per estimated task (a single round: the makespan of a bin is
    // quantised in units of one task = one chunk's serial decode); otherwise plan_serial_grids splits the blocks.
    // Pages cut at restart points (skip_kernels.cuh): a chunk of 32 whole pages is one serial task of ~1000 rows; with
    // few selected pages that chain is the scan's makespan, and with many the makespan is still quantised in chunk
    // times. Cut the pages of the simple8b / gorilla bins into parts so that the scan has about PARTS_TARGET chunks
    // per resident warp (more parts = shorter chains, but one more page open + two more run flushes per part).
    // With every bin at 4 CTAs per SM, 8 chunks per resident warp measured best on C4 (H100: 4 parts of 256 rows per
    // 1000-row page instead of 3 uneven parts of 384 / 384 / 232 rows at a target of 4; DESIGN.md §5).
    uint32_t parts[N_BINS];
    for (int b = 0; b < N_BINS; b++) parts[b] = 1;
    if (pages->d_skip && !s->has_sel) {
      double est_chunks = 0;
      for (int b = 0; b < N_BINS; b++) est_chunks += std::ceil((pages->h_bin_start[b + 1] - pages->h_bin_start[b]) * sel_frac / 32.0);
      const double resident_warps = (double)ctx->sm_count * SCAN_MIN_BLOCKS * (SCAN_THREADS / 32);
      const char *pt_env = getenv("TSKV_PARTS_TARGET");
      uint32_t want = plan_parts_wanted(est_chunks, resident_warps, pt_env ? atof(pt_env) : 8.0);
      const char *parts_env = getenv("TSKV_PARTS");  // fixed number of parts (1 = never cut)
      if (parts_env) want = (uint32_t)std::max(1, atoi(parts_env));
      for (int b = 0; b < N_BINS; b++) {
        const int sb = serial_bin_of(b);
        if (sb / N_VK == TK_GEN || sb % N_VK == VK_GEN) continue;
        uint32_t want_b = want;
        if (sb / N_VK == TK_S8B) {  // TSKV_PARTS_TS: another number of parts for the simple8b-timestamp bins (their rows cost
          // ~1.6 x the rows of RLE-timestamp pages; H100, C4: twice the parts changes nothing, 1.03-1.05 vs 1.02 ms per scan)
          const char *ts_env = getenv("TSKV_PARTS_TS");
          if (ts_env) want_b = (uint32_t)std::max(1, atoi(ts_env));
        }
        uint32_t part_rows = 0;
        parts[b] = plan_bin_parts(pages->h_bin_maxrows[b], SKIP_ROWS, want_b, &part_rows);
        P.bin_parts[b] = parts[b];
        P.bin_part_rows[b] = part_rows;
      }
    }
    double need_sum = 0, occ_weighted = 0;
    int need[N_BINS] = {0}, occ_bin[N_BINS] = {0};
    for (int b = 0; b < N_BINS; b++) {
      uint32_t n_bin = pages->h_bin_start[b + 1] - pages->h_bin_start[b];
      if (!n_bin) continue;
      int occ = 0;
      const int sb = serial_bin_of(b);
      const void *fn = (const void *)(s->has_sel ? scan_kernel_for<true>(sb) : scan_kernel_for<false>(sb, pages->h_bin_narrow[b]));
      cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, fn, SCAN_THREADS, serial_smem_bytes(sb, P.smem_words, P.has_tomb));
      occ = std::max(1, occ);
      occ_bin[b] = occ;
      s->occ[b] = occ;
      const double est_items = n_bin * sel_frac * 1.02 + 32;
      const uint32_t per_task = 32;  // pages per warp task: one chunk
      const double tasks = est_items / per_task * parts[b];
      need[b] = (int)(tasks / (SCAN_THREADS / 32)) + 1;
      need[b] = std::min(need[b], (int)(((uint64_t)(n_bin + per_task - 1) / per_task * parts[b] + SCAN_THREADS / 32 - 1) / (SCAN_THREADS / 32)));
      need_sum += need[b];
      occ_weighted += (double)need[b] * occ;
    }
    const double capacity = need_sum > 0 ? (occ_weighted / need_sum) * ctx->sm_count : 0;  // resident blocks, mixed kernels
    if (need_sum <= capacity) {
      for (int b = 0; b < N_BINS; b++)
        if (need[b]) s->grid[b] = std::max(1, need[b]);
    } else {
      // a chunk of 32 pages is one long serial task, so a bin's time is quantised in rounds of its chunk time - choose
      // the grids that minimise the makespan (plan_serial_grids)
      double chunks[N_BINS], t_chunk[N_BINS];
      for (int b = 0; b < N_BINS; b++) {
        const uint32_t n_bin = pages->h_bin_start[b + 1] - pages->h_bin_start[b];
        chunks[b] = need[b] ? std::ceil((n_bin * sel_frac * 1.02 + 16) / 32.0) * parts[b] : 0;
        // (+ 12 rows' worth per chunk for opening its pages)
        t_chunk[b] = n_bin ? chunk_cost(b) * ((double)pages->h_bin_rows[b] / n_bin / parts[b] + 12.0) : 1.0;
      }
      plan_serial_grids(N_BINS, chunks, t_chunk, occ_bin, ctx->sm_count, SCAN_THREADS / 32, s->grid);
      for (int b = 0; b < N_BINS; b++) s->grid[b] = std::min(s->grid[b], std::max(need[b], 0));
      // TSKV_GRID_OVERSUB=f: f x the planned blocks per bin; the blocks that are not resident at first start as the
      // bins that finish early retire theirs and pick up what is left of the slower bins' chunks
      // H100, C4 at N = 1 (pages cut in 3 parts), ms per scan: planned grids 1.43-1.50, 2 x 1.10, 4 x 1.02 = one warp per
      // chunk 1.02-1.03. Uncut pages too: planned grids 1.26-1.34, 4 x 1.12; FIRST / LAST scans (C5 shape) and
      // host-resident page sets are the same with either (31.0-31.7 ms).
      {
        const char *ov = getenv("TSKV_GRID_OVERSUB");
        const double f = ov ? atof(ov) : 4.0;
        if (f > 1.0)
          for (int b = 0; b < N_BINS; b++) s->grid[b] = std::min(std::max(need[b], 0), (int)std::ceil(s->grid[b] * f));
      }
      // TSKV_GRID_MODE=1: one warp per chunk for every bin; the block scheduler queues what does not fit
      const char *gm = getenv("TSKV_GRID_MODE");
      if (gm && gm[0] == '1')
        for (int b = 0; b < N_BINS; b++) s->grid[b] = need[b];
    }
  }
  // ---- merge pass over the overlapping chunks (merge_kernels.cuh): which merge column groups this scan reads
  // (series selected, not pruned by its time bounds), and the field pages of the query's columns to decode for them
  s->chunk_epoch = pages->chunk_epoch;
  if (pages->merge_rows) {
    const OverlapPlan &op = pages->overlap;
    const size_t n_mcg = op.mcg_cg.size();
    std::vector<uint8_t> active(n_mcg, 0);
    std::vector<uint32_t> mpage;
    std::vector<uint64_t> mrow_off, mbm_off;
    for (size_t k = 0; k < n_mcg; k++) {
      const uint32_t cg = op.mcg_cg[k], tp = pages->h_cg_time_page[cg];
      const tskv_page_desc &td = pages->h_descs[tp];
      if (q->series_ids && !std::binary_search(q->series_ids, q->series_ids + q->n_series, td.series_id)) continue;
      if (q->n_time_ranges) {  // filter_column_groups (reader/chunk.rs:12-50)
        bool overlaps = false;
        for (uint32_t r = 0; r < q->n_time_ranges; r++)
          overlaps = overlaps || (pages->h_cg_bounds[cg].min_ts <= q->time_ranges[r].max_ts && pages->h_cg_bounds[cg].max_ts >= q->time_ranges[r].min_ts);
        if (!overlaps) continue;
      }
      bool any = false;
      for (uint64_t p = (uint64_t)tp + 1; p < pages->n_descs && pages->h_descs[p].phys_type != TSKV_PT_TIME; p++)
        for (uint32_t c = 0; c < q->n_columns; c++)
          if (pages->h_descs[p].column_id == q->columns[c].column_id) {
            if (pages->h_descs[p].phys_type != q->columns[c].phys_type) {
              ctx->set_error("page type does not match the query column type", (int64_t)p);
              free_scan(s);
              return TSKV_ERR_INVALID_ARG;
            }
            any = true;
            mpage.push_back((uint32_t)p);
            mrow_off.push_back((uint64_t)c * pages->merge_rows + op.mcg_row0[k]);
            mbm_off.push_back(((uint64_t)c * pages->merge_bm_words + pages->h_mcg_bm0[k]) * 4);
            s->merge_page_bytes += pages->h_descs[p].size;
          }
      if (!any) continue;  // a column group without any projected column yields no batch (column_group/mod.rs:43-52)
      active[k] = 1;
      s->merge_page_bytes += td.size;
      s->merge_read_pages++;
    }
    s->n_merge_pages = (uint32_t)mpage.size();
    s->merge_read_pages += mpage.size();
    cudaError_t me = stream_alloc(ctx, &s->d_mcg_active, n_mcg);
    if (me == cudaSuccess) me = cudaMemcpyAsync(s->d_mcg_active, active.data(), n_mcg, cudaMemcpyHostToDevice, ctx->stream);
    if (me == cudaSuccess) me = stream_alloc(ctx, &s->d_mvals, (size_t)q->n_columns * pages->merge_rows);
    if (me == cudaSuccess) me = stream_alloc(ctx, &s->d_mvalid, (size_t)q->n_columns * pages->merge_bm_words);
    if (me == cudaSuccess) me = stream_alloc(ctx, &s->d_mpage, mpage.size());
    if (me == cudaSuccess) me = stream_alloc(ctx, &s->d_mrow_off, mpage.size());
    if (me == cudaSuccess) me = stream_alloc(ctx, &s->d_mbm_off, mpage.size());
    if (me == cudaSuccess && !mpage.empty()) {
      me = cudaMemcpyAsync(s->d_mpage, mpage.data(), mpage.size() * 4, cudaMemcpyHostToDevice, ctx->stream);
      if (me == cudaSuccess) me = cudaMemcpyAsync(s->d_mrow_off, mrow_off.data(), mpage.size() * 8, cudaMemcpyHostToDevice, ctx->stream);
      if (me == cudaSuccess) me = cudaMemcpyAsync(s->d_mbm_off, mbm_off.data(), mpage.size() * 8, cudaMemcpyHostToDevice, ctx->stream);
    }
    if (me == cudaSuccess) me = cudaStreamSynchronize(ctx->stream);  // the host vectors go out of scope
    if (me != cudaSuccess) {
      ctx->set_error(std::string("scan_prepare (merge pass): ") + cudaGetErrorString(me));
      free_scan(s);
      return me == cudaErrorMemoryAllocation ? TSKV_ERR_OOM : TSKV_ERR_CUDA;
    }
    h2d += n_mcg + mpage.size() * 20;
    MergeParams &M = s->merge;
    M.ts = pages->d_merge_ts;
    M.mcg_row0 = pages->d_mcg_row0;
    M.mcg_cg = pages->d_mcg_cg;
    M.mcg_stream = pages->d_mcg_stream;
    M.stream_group = pages->d_stream_group;
    M.stream_first_mcg = pages->d_stream_first_mcg;
    M.group_first_stream = pages->d_group_first_stream;
    M.mcg_active = s->d_mcg_active;
    M.vals = s->d_mvals;
    M.valid = s->d_mvalid;
    M.mcg_bm0 = pages->d_mcg_bm0;
    M.cg_time_page = pages->d_cg_time_page;
    M.cg_slot = s->d_cg_slot;
    M.n_rows = pages->merge_rows;
    M.bm_words = pages->merge_bm_words;
    M.n_mcg = (uint32_t)n_mcg;
    M.sel = s->has_sel ? 1u : 0u;
  }
  ctx->counters.h2d_bytes = h2d;
  *out_scan = s;
  return TSKV_OK;
}

tskv_status tskvgpu_scan_prepare(tskv_ctx *ctx, const tskv_pages *pages, const tskv_query *q, tskv_scan **out_scan) {
  return prepare_scan(ctx, pages, q, 0, TagGroups{}, out_scan);
}

static tskv_status prepare_sliding(tskv_ctx *ctx, const tskv_pages *pages, const tskv_query *q, int64_t slide,
                                   const TagGroups &tg, tskv_scan **out_scan) {
  if (!ctx || !pages || !q || !out_scan) return TSKV_ERR_INVALID_ARG;
  if (slide <= 0 || q->width <= 0) {
    std::lock_guard<std::mutex> lock(ctx->mu);
    ctx->set_error("sliding windows: slide and window must be > 0");
    *out_scan = nullptr;
    return TSKV_ERR_INVALID_ARG;
  }
  return prepare_scan(ctx, pages, q, slide == q->width ? 0 : slide, tg, out_scan);  // slide == window: a tumbling window
}

tskv_status tskvgpu_scan_prepare_sliding(tskv_ctx *ctx, const tskv_pages *pages, const tskv_query *q, int64_t slide,
                                         tskv_scan **out_scan) {
  return prepare_sliding(ctx, pages, q, slide, TagGroups{}, out_scan);
}

tskv_status tskvgpu_scan_prepare_grouped(tskv_ctx *ctx, const tskv_pages *pages, const tskv_query *q, const uint32_t *group_ids,
                                         uint32_t n_groups, int64_t slide, tskv_scan **out_scan) {
  const TagGroups tg{true, group_ids, n_groups};
  return slide ? prepare_sliding(ctx, pages, q, slide, tg, out_scan) : prepare_scan(ctx, pages, q, 0, tg, out_scan);
}

// Enqueues one full pass on the context stream, no host synchronisation:
//   selection -> compacted work list -> (host-resident arenas: PCIe gather of the selected pages)
//   -> state init -> one fused decode/filter/reduce kernel per decode-kind bin -> export.
// `capturing`: the calls are being recorded into a CUDA graph - timing events are left out (only the fork / join / gather
// dependencies are recorded, on events created without timing).
static tskv_status enqueue_scan(tskv_ctx *ctx, tskv_scan *s, bool capturing = false) {
  const tskv_pages *pages = s->pages;
  const uint32_t n_items = pages->n_items;
  if (s->tomb_epoch != pages->tomb_epoch) {
    ctx->set_error("the page set's tombstones changed after this scan was prepared", -1);
    return TSKV_ERR_INVALID_ARG;
  }
  if (s->chunk_epoch != pages->chunk_epoch) {
    ctx->set_error("the page set's chunk files changed after this scan was prepared", -1);
    return TSKV_ERR_INVALID_ARG;
  }
  if (!capturing) cudaEventRecord(s->ev0, ctx->stream);
  unsigned long long *aux = reinterpret_cast<unsigned long long *>(s->d_task_counter);
  uint64_t launches = 0;
  {  // state identities + the pass's scratch (task counters / status / counters, bin starts, work-list buckets): one launch
    const uint32_t init_blocks = (uint32_t)std::min<uint64_t>((s->kern_sl.total + 255) / 256, 4096);
    k_init_state<<<std::max(1u, init_blocks), 256, 0, ctx->stream>>>(s->params.state, s->kern_sl, aux, 32, s->d_bin_cstart, N_BINS + 2,
                                                                   s->d_bucket, N_BINS * s->n_cols * WL_SUB);
    launches++;
  }
  // slot of every column group: the row filter, the merge pass and the item-driven work list need it per GROUP; the
  // selection-driven work list finds a selected series' groups itself
  const bool need_cg_slot = s->worklist_by_items || s->preds.n || (s->merge.n_rows && s->n_merge_pages);
  if (pages->n_cg && need_cg_slot) {
    if (s->d_rank_slot) {
      CU_TRY(ctx, cudaMemsetAsync(s->d_rank_slot, 0xff, pages->series.size() * 4, ctx->stream));
      if (s->n_series_sel) {
        k_select_ids<<<(s->n_series_sel + 255) / 256, 256, 0, ctx->stream>>>(pages->d_series_sorted, (uint32_t)pages->series.size(), s->d_series,
                                                                         s->n_series_sel, s->d_rank_slot);
        launches++;
      }
    }
    k_select_cg<<<(pages->n_cg + 255) / 256, 256, 0, ctx->stream>>>(pages->n_cg, s->d_rank_slot, pages->d_cg_series_rank, s->d_cg_slot);
    launches++;
  }
  if (s->preds.n && pages->n_cg) {  // row filter: keep bits of every selected column group (host-resident pages: read in place)
    k_row_filter<<<(pages->n_cg + 127) / 128, 128, 0, ctx->stream>>>(pages->h_mapped ? pages->h_mapped : pages->d_arena, pages->d_descs,
                                                                     pages->n_descs, pages->d_cg_time_page, pages->n_cg, s->d_cg_slot,
                                                                     s->preds, pages->d_keep_off, s->d_row_keep, s->d_status, s->d_err_page);
    launches++;
  }
  if (n_items && s->worklist_by_items) {
    k_flag_items<<<s->n_blocks, 1024, 0, ctx->stream>>>(pages->d_descs, pages->d_item_info,
                                                        pages->d_cg_time_page, n_items, s->d_cg_slot, s->d_cols,
                                                        s->n_cols, pages->d_bin_start, s->d_item_flag,
                                                        s->d_block_count, s->d_counters, s->d_status,
                                                        s->prune.n ? pages->d_cg_bounds : nullptr, s->prune, pages->d_cg_merge,
                                                        s->preds.n ? pages->d_page_stats : nullptr, s->preds, pages->n_descs, pages->n_cg);
    k_scan_blocks<<<1, 1024, 0, ctx->stream>>>(s->d_block_count, s->n_blocks, s->d_bin_cstart + N_BINS + 1);
    k_scatter_items<<<s->n_blocks, 1024, 0, ctx->stream>>>(pages->d_item_page, pages->d_item_cg, n_items, s->d_item_flag,
                                                           s->d_block_count, s->d_cg_slot, pages->d_bin_start,
                                                           s->d_work_page, s->d_work_slot, s->d_work_qcol,
                                                           s->d_bin_cstart, s->d_bin_cstart + N_BINS + 1);
    launches += 3;
  } else if (n_items) {
    WorkListArgs A{};
    A.descs = pages->d_descs;
    A.n_descs = pages->n_descs;
    A.cg_time_page = pages->d_cg_time_page;
    A.n_cg = pages->n_cg;
    A.rank_cg_start = pages->d_rank_cg_start;
    A.rank_cg = pages->d_rank_cg;
    A.page_bin = pages->d_page_bin;
    // narrow pages apart only where a bin holds both kinds (NARROW_SOME kernels choose per chunk)
    A.page_narrow = std::any_of(pages->h_bin_narrow, pages->h_bin_narrow + N_BINS, [](uint8_t m) { return m == NARROW_SOME; })
                        ? pages->d_narrow : nullptr;
    A.set_series = pages->d_series_sorted;
    A.n_set_series = (uint32_t)pages->series.size();
    A.series_ids = s->d_series;
    A.n_sel = s->d_series ? s->n_series_sel : (uint32_t)pages->series.size();
    A.walk = s->d_walk;
    A.cols = s->d_cols;
    A.n_cols = s->n_cols;
    A.cg_bounds = s->prune.n ? pages->d_cg_bounds : nullptr;
    A.prune = s->prune;
    A.cg_merge = pages->d_cg_merge;
    A.page_stats = s->preds.n ? pages->d_page_stats : nullptr;
    A.preds = s->preds;
    const uint32_t n_buckets = N_BINS * s->n_cols * WL_SUB;
    A.bucket_count = s->d_bucket;
    A.bucket_off = s->d_bucket + n_buckets;
    A.work_page = s->d_work_page;
    A.work_slot = s->d_work_slot;
    A.work_qcol = s->d_work_qcol;
    A.counters = s->d_counters;
    A.status = s->d_status;
    const uint32_t wblocks = std::max(1u, (A.n_sel + WL_THREADS - 1) / WL_THREADS);
    if (A.n_sel) k_worklist_count<<<wblocks, WL_THREADS, n_buckets * 4, ctx->stream>>>(A);
    k_worklist_offsets<<<1, 256, 0, ctx->stream>>>(s->d_bucket, s->d_bucket + n_buckets, s->n_cols * WL_SUB, s->d_bin_cstart);
    if (A.n_sel) k_worklist_emit<<<wblocks, WL_THREADS, 2 * n_buckets * 4, ctx->stream>>>(A);
    launches += 3;
  }
  if (s->merge.n_rows && s->n_merge_pages) {  // overlapping chunks: decode the query's columns, merge + aggregate per row
    CU_TRY(ctx, cudaMemsetAsync(s->d_mvalid, 0, (size_t)s->n_cols * s->merge.bm_words * 4, ctx->stream));
    const uint32_t dblocks = (uint32_t)(((uint64_t)s->n_merge_pages * 32 + DECODE_THREADS - 1) / DECODE_THREADS);
    k_decode_warp<<<dblocks, DECODE_THREADS, 0, ctx->stream>>>(pages->h_mapped ? pages->h_mapped : pages->d_arena, pages->d_descs, 0, s->d_mpage,
                                                              s->n_merge_pages, s->d_mrow_off, s->d_mbm_off, s->d_mvals,
                                                              reinterpret_cast<uint8_t *>(s->d_mvalid), s->d_status, s->d_err_page, s->d_stats);
    const uint32_t mblocks = (uint32_t)((s->merge.n_rows + 127) / 128);
    k_merge_chunks<<<mblocks, 128, 0, ctx->stream>>>(s->params, s->merge);
    launches += 2;
  }
  cudaEvent_t ev_fork = capturing ? s->ev_cfork : s->ev_bin[0];
  cudaEventRecord(ev_fork, ctx->stream);  // fork
  // Host-resident pages: one bin's gather already saturates PCIe, so the gathers are chained largest bin first
  // (an event per bin); each bin's CRC check and scan then overlap the next bins' transfers and only the smallest
  // bin's tail is exposed after the last byte has arrived.
  int order[N_BINS];
  for (int b = 0; b < N_BINS; b++) order[b] = b;
  static const bool gather_concurrent = getenv("TSKV_GATHER_CONCURRENT") != nullptr;
  if (pages->h_mapped && !gather_concurrent)
    std::stable_sort(order, order + N_BINS, [&](int a, int b) { return pages->h_bin_bytes[a] > pages->h_bin_bytes[b]; });
  else if (!pages->h_mapped)
    std::stable_sort(order, order + N_BINS, [&](int a, int b) { return chunk_cost(a) > chunk_cost(b); });
  int prev_gather = -1;
  bool crc_forked = false;
  for (int oi = 0; oi < N_BINS; oi++) {
    const int b = order[oi];
    if (!s->grid[b]) continue;
    cudaStreamWaitEvent(ctx->bin_stream[b], ev_fork, 0);
    int bin = b;
    if (pages->h_mapped) {
      if (prev_gather >= 0 && !gather_concurrent) cudaStreamWaitEvent(ctx->bin_stream[b], s->ev_gather[prev_gather], 0);
      uint32_t n_bin = pages->h_bin_start[b + 1] - pages->h_bin_start[b];
      uint32_t gblocks = std::max(1u, std::min<uint32_t>((uint32_t)ctx->sm_count * 4, (n_bin + 7) / 8));
      k_gather_pages<<<gblocks, 256, 0, ctx->bin_stream[b]>>>(pages->h_mapped, pages->d_arena, pages->d_descs,
                                                              pages->d_time_page_of, s->d_work_page, s->d_work_qcol,
                                                              s->d_bin_cstart, bin);
      launches++;
      cudaEventRecord(s->ev_gather[b], ctx->bin_stream[b]);
      prev_gather = b;
    }
    if (pages->verify_on_read) {  // Page::crc_validation on every read (tsm/reader.rs:259), also for pages resident in HBM
      uint32_t n_bin = pages->h_bin_start[b + 1] - pages->h_bin_start[b];
      // In front of the bin's fused kernel (HBM-resident pages) / after the bin's transfer, under the next bin's
      // (host-resident pages). TSKV_CRC_CONCURRENT=1 runs the checks of HBM-resident pages BESIDE the fused kernels on a
      // stream of their own instead - H100, C4: 1.84-2.03 ms per scan with 1-8 CRC blocks per SM against
      // 1.39 ms in line (the check needs the whole machine's lanes to hide its dependent table lookups; a slice of the
      // machine makes it the step's critical path). A mismatch is reported in its own status slot either way and outranks
      // whatever the decoders made of the corrupt page.
      const bool crc_concurrent = !pages->h_mapped && getenv("TSKV_CRC_CONCURRENT") != nullptr;
      if (!crc_concurrent) {
        uint32_t gblocks = std::max(1u, std::min<uint32_t>((uint32_t)ctx->sm_count * 4, (n_bin + 7) / 8));
        k_verify_crc<<<gblocks, 256, 0, ctx->bin_stream[b]>>>(pages->d_arena, pages->d_descs, pages->d_time_page_of,
                                                              s->d_work_page, s->d_work_qcol, s->d_bin_cstart, bin,
                                                              pages->d_crc_tables, s->d_crc_status, s->d_crc_err_page);
      } else {
        if (!crc_forked) cudaStreamWaitEvent(ctx->crc_stream, ev_fork, 0);
        crc_forked = true;
        const char *bps_env = getenv("TSKV_CRC_BLOCKS_PER_SM");
        const uint32_t bps = bps_env ? (uint32_t)std::max(1, atoi(bps_env)) : 1u;
        uint32_t gblocks = std::max(1u, std::min<uint32_t>((uint32_t)ctx->sm_count * bps, (n_bin + 255) / 256));
        k_verify_crc<<<gblocks, 256, 0, ctx->crc_stream>>>(pages->d_arena, pages->d_descs, pages->d_time_page_of,
                                                           s->d_work_page, s->d_work_qcol, s->d_bin_cstart, bin,
                                                           pages->d_crc_tables, s->d_crc_status, s->d_crc_err_page);
      }
      launches++;
    }
    if (!capturing) cudaEventRecord(s->ev_bin_start[b], ctx->bin_stream[b]);
    const int sb = serial_bin_of(b);
    void *args[] = {(void *)&s->params, (void *)&bin};
    const void *fn = (const void *)(s->has_sel ? scan_kernel_for<true>(sb) : scan_kernel_for<false>(sb, pages->h_bin_narrow[b]));
    CU_TRY(ctx, cudaLaunchKernel(fn, dim3(s->grid[b]), dim3(SCAN_THREADS), args, serial_smem_bytes(sb, s->params.smem_words, s->params.has_tomb),
                                 ctx->bin_stream[b]));
    cudaEvent_t ev_done = capturing ? s->ev_cjoin[b] : s->ev_bin_done[b];
    cudaEventRecord(ev_done, ctx->bin_stream[b]);
    cudaStreamWaitEvent(ctx->stream, ev_done, 0);  // join
    launches++;
  }
  if (crc_forked) {  // join the concurrent CRC checks
    cudaEvent_t ev = capturing ? s->ev_ccrc : s->ev_crc;
    cudaEventRecord(ev, ctx->crc_stream);
    cudaStreamWaitEvent(ctx->stream, ev, 0);
  }
  if (!capturing) cudaEventRecord(s->ev_bin[N_BINS], ctx->stream);
  if (s->n_combine) {  // sliding windows: every window folds its panes (it writes every array the kernels fill)
    const uint32_t bx = (uint32_t)std::min<uint64_t>((s->layout.n_cells + 255) / 256, 1024);
    k_window_combine<<<dim3(std::max(1u, bx), s->n_combine), 256, 0, ctx->stream>>>(
        s->d_pane_state, s->d_state, s->d_combine, (uint32_t)s->layout.n_groups, s->n_windows, s->n_panes, s->win_k);
    launches++;
  }
  if (s->has_sel || s->n_means) {
    uint64_t work = std::max(std::max(s->sl.first_cells, s->sl.last_cells), s->n_means ? s->layout.n_cells : 0);
    uint32_t b = (uint32_t)std::min<uint64_t>((work + 255) / 256, 4096);
    k_export_pairs<<<std::max(1u, b), 256, 0, ctx->stream>>>(s->d_state, s->sl, s->d_means, s->n_means, s->layout.n_cells);
    launches++;
  }
  if (!capturing) cudaEventRecord(s->ev1, ctx->stream);
  CU_TRY(ctx, cudaGetLastError());
  ctx->counters.kernel_launches = launches;
  s->enqueued = true;
  return TSKV_OK;
}

// Waits for the stream, surfaces device-side decode errors and refreshes the counters.
static tskv_status sync_scan(tskv_ctx *ctx, tskv_scan *s) {
  tskv_status st = fetch_status(ctx, s->d_crc_status, s->d_crc_err_page);  // Page::crc_validation comes first (tsm/reader.rs:259)
  if (st == TSKV_OK) st = fetch_status(ctx, s->d_status, s->d_err_page);
  if (st != TSKV_OK) {
    if (st == TSKV_ERR_INVALID_ARG) ctx->set_error("page type does not match the query column type", ctx->err_page);
    return st;
  }
  unsigned long long aux[5 + N_BINS] = {0};  // stats[2], pages, bytes, per-bin bytes[N_BINS], pruned pages
  CU_TRY(ctx, cudaMemcpy(aux, s->d_stats, (5 + N_BINS) * 8, cudaMemcpyDeviceToHost));
  ctx->counters.pruned_page_count = aux[4 + N_BINS];
  float ms = 0;
  cudaEventElapsedTime(&ms, s->ev0, s->ev1);
  ctx->counters.elapsed_scan_ms = ms;
  ctx->counters.points_decoded = aux[0];
  ctx->counters.rows_in_range = aux[1];
  ctx->counters.page_read_count = aux[2] + s->merge_read_pages;
  ctx->counters.page_read_bytes = aux[3] + s->merge_page_bytes;
  float fused = 0;
  cudaEventElapsedTime(&fused, s->ev_bin[0], s->ev_bin[N_BINS]);
  ctx->counters.elapsed_fused_ms = fused;
  ctx->counters.dominant_kernel_ms = 0;
  ctx->counters.dominant_kernel_bytes = 0;
  ctx->counters.dominant_kernel_bin = 0;
  if (getenv("TSKV_DEBUG_BINS")) {  // (events of the un-captured pass: meaningful with TSKV_NO_GRAPH=1)
    float pro = 0, epi = 0;
    cudaEventElapsedTime(&pro, s->ev0, s->ev_bin[0]);
    cudaEventElapsedTime(&epi, s->ev_bin[N_BINS], s->ev1);
    fprintf(stderr, "[tskv] prologue (select, work list, init%s) %.3f ms, fused %.3f ms, epilogue %.3f ms\n",
            s->merge.n_rows ? ", merge pass" : "", pro, fused, epi);
  }
  for (int b = 0; b < N_BINS; b++) {
    if (!s->grid[b]) continue;
    float t = 0;
    cudaEventElapsedTime(&t, s->ev_bin_start[b], s->ev_bin_done[b]);
    if (getenv("TSKV_DEBUG_BINS")) {
      float t0 = 0;
      cudaEventElapsedTime(&t0, s->ev_bin[0], s->ev_bin_start[b]);
      fprintf(stderr, "[tskv] bin %d grid %d, %d CTAs/SM: start +%.3f ms, run %.3f ms, %llu bytes\n", b,
              s->grid[b], s->occ[b], t0, t, aux[4 + b]);
    }
    if (t > ctx->counters.dominant_kernel_ms) {
      ctx->counters.dominant_kernel_ms = t;
      ctx->counters.dominant_kernel_bytes = aux[4 + b];
      ctx->counters.dominant_kernel_bin = (uint64_t)b;
    }
  }
  return TSKV_OK;
}

tskv_status tskvgpu_scan_enqueue(tskv_ctx *ctx, tskv_scan *s) {
  if (!ctx || !s) return TSKV_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(ctx->mu);
  cudaSetDevice(ctx->device);
  static const bool no_graph = getenv("TSKV_NO_GRAPH") != nullptr;
  s->n_enqueued++;
  if (no_graph || s->graph_failed || s->n_enqueued < 2) return enqueue_scan(ctx, s);
  if (!s->graph_exec) {
    cudaGraph_t graph = nullptr;
    if (!s->ev_cfork) {
      cudaEventCreateWithFlags(&s->ev_cfork, cudaEventDisableTiming);
      for (int b = 0; b < N_BINS; b++) cudaEventCreateWithFlags(&s->ev_cjoin[b], cudaEventDisableTiming);
    }
    bool ok = cudaStreamBeginCapture(ctx->stream, cudaStreamCaptureModeThreadLocal) == cudaSuccess;
    if (ok) {
      const tskv_status st = enqueue_scan(ctx, s, true);  // the bin streams join the capture through the fork event
      const cudaError_t e = cudaStreamEndCapture(ctx->stream, &graph);
      ok = st == TSKV_OK && e == cudaSuccess && graph && cudaGraphInstantiate(&s->graph_exec, graph, 0) == cudaSuccess;
      if (graph) cudaGraphDestroy(graph);
    }
    if (!ok) {  // anything the capture did not like: replay the pass call by call, as before
      if (getenv("TSKV_DEBUG_BINS")) fprintf(stderr, "[tskv] graph capture failed (%s): direct launches\n", cudaGetErrorString(cudaGetLastError()));
      cudaGetLastError();
      s->graph_exec = nullptr;
      s->graph_failed = true;
      return enqueue_scan(ctx, s);
    }
  }
  CU_TRY(ctx, cudaGraphLaunch(s->graph_exec, ctx->stream));
  s->enqueued = true;
  return TSKV_OK;
}

tskv_status tskvgpu_scan_sync(tskv_ctx *ctx, tskv_scan *s) {
  if (!ctx || !s || !s->enqueued) return TSKV_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(ctx->mu);
  cudaSetDevice(ctx->device);
  return sync_scan(ctx, s);
}

tskv_status tskvgpu_scan_run(tskv_ctx *ctx, tskv_scan *s) {
  if (!ctx || !s) return TSKV_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(ctx->mu);
  cudaSetDevice(ctx->device);
  tskv_status st = enqueue_scan(ctx, s);
  if (st != TSKV_OK) return st;
  return sync_scan(ctx, s);
}

tskv_status tskvgpu_scan_partials(tskv_ctx *ctx, tskv_scan *s, tskv_partials_view *out) {
  if (!ctx || !s || !out) return TSKV_ERR_INVALID_ARG;
  const StateLayout &L = s->sl;
  uint64_t base = (uint64_t)(uintptr_t)s->d_state;
  out->sum_i64_ptr = base + L.sum_i64_off * 8;
  out->sum_i64_len = L.sum_i64_len;
  out->sum_f64_ptr = base + L.sum_f64_off * 8;
  out->sum_f64_len = L.sum_f64_len;
  out->min_i64_ptr = base + L.min_off * 8;
  out->min_i64_len = L.min_len;
  out->max_i64_ptr = base + L.max_off * 8;
  out->max_i64_len = L.max_len;
  out->sel_val_ptr = base + L.selval_off * 8;
  out->sel_val_len = L.selval_len;
  out->sel_first_len = L.first_cells;
  out->sel_last_len = L.last_cells;
  return TSKV_OK;
}

tskv_status tskvgpu_scan_exchange_view(tskv_ctx *ctx, tskv_scan *s, uint64_t *out_dptr, uint64_t *out_words) {
  if (!ctx || !s || !out_dptr || !out_words) return TSKV_ERR_INVALID_ARG;
  *out_dptr = (uint64_t)(uintptr_t)s->d_state;
  *out_words = s->sl.selval_off + s->sl.selval_len;  // sum_i64 | sum_f64 | min+first keys | max+last keys | values
  return TSKV_OK;
}

tskv_status tskvgpu_scan_merge_gathered(tskv_ctx *ctx, tskv_scan *s, uint64_t gathered_dptr, uint32_t n_ranks) {
  if (!ctx || !s || !gathered_dptr || n_ranks == 0) return TSKV_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(ctx->mu);
  cudaSetDevice(ctx->device);
  const uint64_t words = s->sl.selval_off + s->sl.selval_len;
  uint32_t blocks = (uint32_t)std::min<uint64_t>((words + 255) / 256, 2048);
  k_merge_gathered<<<std::max(1u, blocks), 256, 0, ctx->stream>>>(s->d_state, s->sl, reinterpret_cast<const uint64_t *>((uintptr_t)gathered_dptr),
                                                                   n_ranks, words);
  CU_TRY(ctx, cudaGetLastError());
  return TSKV_OK;
}

tskv_status tskvgpu_scan_exchange(tskv_ctx *ctx, tskv_scan *s) {
  if (!ctx || !s) return TSKV_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(ctx->mu);
  cudaSetDevice(ctx->device);
  if (!ctx->comm) {
    ctx->set_error("tskvgpu_scan_exchange: no communicator (tskvgpu_comm_init)");
    return TSKV_ERR_NCCL;
  }
  const NcclApi &N = nccl_api();
  const uint64_t words = s->sl.selval_off + s->sl.selval_len;  // sum_i64 | sum_f64 | min+first keys | max+last keys | values
  if (!s->d_gathered) CU_TRY(ctx, stream_alloc(ctx, &s->d_gathered, (size_t)ctx->n_ranks * words));
  const ncclResult_t r = N.AllGather(s->d_state, s->d_gathered, words, ncclUint64, ctx->comm, ctx->stream);
  if (r != ncclSuccess) {
    ctx->set_error(std::string("ncclAllGather: ") + N.GetErrorString(r));
    return TSKV_ERR_NCCL;
  }
  uint32_t blocks = (uint32_t)std::min<uint64_t>((words + 255) / 256, 2048);
  k_merge_gathered<<<std::max(1u, blocks), 256, 0, ctx->stream>>>(s->d_state, s->sl, s->d_gathered, (uint32_t)ctx->n_ranks, words);
  CU_TRY(ctx, cudaGetLastError());
  return TSKV_OK;
}

tskv_status tskvgpu_scan_snapshot_keys(tskv_ctx *ctx, tskv_scan *s) {
  if (!ctx || !s) return TSKV_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(ctx->mu);
  cudaSetDevice(ctx->device);
  if (s->has_sel) {
    k_snapshot_keys<<<256, 256, 0, ctx->stream>>>(s->d_state, s->sl);
    CU_TRY(ctx, cudaGetLastError());
  }
  return TSKV_OK;
}

tskv_status tskvgpu_scan_mask_values(tskv_ctx *ctx, tskv_scan *s) {
  if (!ctx || !s) return TSKV_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(ctx->mu);
  cudaSetDevice(ctx->device);
  if (s->has_sel) {
    k_mask_values<<<256, 256, 0, ctx->stream>>>(s->d_state, s->sl);
    CU_TRY(ctx, cudaGetLastError());
  }
  return TSKV_OK;
}

static tskv_status finalize_device(tskv_ctx *ctx, tskv_scan *s) {
  const tskv_output_layout &L = s->layout;
  dim3 grid((uint32_t)((L.n_cells + 255) / 256), s->n_out);
  k_finalize<<<grid, 256, 0, ctx->stream>>>(s->d_state, s->d_outs, s->n_out, L.n_cells, L.bitmap_stride, s->d_values,
                                            s->d_validity);
  CU_TRY(ctx, cudaGetLastError());
  return TSKV_OK;
}

tskv_status tskvgpu_scan_finalize(tskv_ctx *ctx, tskv_scan *s, uint64_t *out_values, uint8_t *out_validity) {
  if (!ctx || !s || !out_values || !out_validity) return TSKV_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(ctx->mu);
  cudaSetDevice(ctx->device);
  tskv_status st = finalize_device(ctx, s);
  if (st != TSKV_OK) return st;
  CU_TRY(ctx, cudaMemcpyAsync(out_values, s->d_values, s->layout.values_bytes, cudaMemcpyDeviceToHost, ctx->stream));
  CU_TRY(ctx, cudaMemcpyAsync(out_validity, s->d_validity, s->layout.validity_bytes, cudaMemcpyDeviceToHost, ctx->stream));
  CU_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  return TSKV_OK;
}

tskv_status tskvgpu_scan_finalize_device(tskv_ctx *ctx, tskv_scan *s, uint64_t *out_values_dptr,
                                         uint64_t *out_validity_dptr) {
  if (!ctx || !s) return TSKV_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(ctx->mu);
  cudaSetDevice(ctx->device);
  tskv_status st = finalize_device(ctx, s);
  if (st != TSKV_OK) return st;
  if (out_values_dptr) *out_values_dptr = (uint64_t)(uintptr_t)s->d_values;
  if (out_validity_dptr) *out_validity_dptr = (uint64_t)(uintptr_t)s->d_validity;
  return TSKV_OK;
}

void tskvgpu_scan_destroy(tskv_ctx *ctx, tskv_scan *s) {
  if (ctx) cudaSetDevice(ctx->device);
  free_scan(s);
}

static tskv_status scan_aggregate(tskv_ctx *ctx, const tskv_pages *pages, const tskv_query *q, int64_t slide,
                                  const TagGroups &tg, uint64_t *out_values, uint8_t *out_validity) {
  if (!out_values || !out_validity) return TSKV_ERR_INVALID_ARG;
  tskv_scan *s = nullptr;
  tskv_status st = slide ? prepare_sliding(ctx, pages, q, slide, tg, &s) : prepare_scan(ctx, pages, q, 0, tg, &s);
  if (st != TSKV_OK) return st;
  st = tskvgpu_scan_run(ctx, s);
  if (st == TSKV_OK) st = tskvgpu_scan_finalize(ctx, s, out_values, out_validity);
  ctx->counters.kernel_launches += 1;
  tskvgpu_scan_destroy(ctx, s);
  return st;
}

tskv_status tskvgpu_scan_aggregate(tskv_ctx *ctx, const tskv_pages *pages, const tskv_query *q,
                                   uint64_t *out_values, uint8_t *out_validity) {
  return scan_aggregate(ctx, pages, q, 0, TagGroups{}, out_values, out_validity);
}

tskv_status tskvgpu_scan_aggregate_sliding(tskv_ctx *ctx, const tskv_pages *pages, const tskv_query *q, int64_t slide,
                                           uint64_t *out_values, uint8_t *out_validity) {
  if (slide <= 0) {  // (slide 0 would select the tumbling scan)
    if (!ctx) return TSKV_ERR_INVALID_ARG;
    std::lock_guard<std::mutex> lock(ctx->mu);
    ctx->set_error("sliding windows: slide and window must be > 0");
    return TSKV_ERR_INVALID_ARG;
  }
  return scan_aggregate(ctx, pages, q, slide, TagGroups{}, out_values, out_validity);
}

tskv_status tskvgpu_scan_aggregate_grouped(tskv_ctx *ctx, const tskv_pages *pages, const tskv_query *q, const uint32_t *group_ids,
                                           uint32_t n_groups, int64_t slide, uint64_t *out_values, uint8_t *out_validity) {
  return scan_aggregate(ctx, pages, q, slide, TagGroups{true, group_ids, n_groups}, out_values, out_validity);
}

}  // extern "C"
