// tskv_gpu.cu — C-ABI entry points of include/tskv_gpu.h: context, page upload, decode-only and the
// fused scan/aggregate launches. Host logic only; the device code is in scan_kernels.cuh.
#include <algorithm>
#include <cmath>
#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <mutex>
#include <numeric>
#include <string>
#include <thread>
#include <type_traits>
#include <unordered_map>
#include <vector>

#include <cub/device/device_radix_sort.cuh>
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

// Owners of the library's CUDA resources: each handle is released by its deleter when its owner goes away or is
// replaced.
struct DevFree {
  void operator()(void *p) const { cudaFree(p); }
};
struct AsyncFree {  // stream-ordered: the buffer returns to the pool after the work enqueued before the free
  cudaStream_t stream = nullptr;
  void operator()(void *p) const { cudaFreeAsync(p, stream); }
};
struct EventDestroy {
  void operator()(cudaEvent_t e) const { cudaEventDestroy(e); }
};
struct StreamDestroy {
  void operator()(cudaStream_t st) const { cudaStreamDestroy(st); }
};
struct GraphExecDestroy {
  void operator()(cudaGraphExec_t g) const { cudaGraphExecDestroy(g); }
};
struct HostUnregister {
  void operator()(void *p) const { cudaHostUnregister(p); }
};
template <typename T>
using dev_ptr = std::unique_ptr<T[], DevFree>;
template <typename T>
using async_ptr = std::unique_ptr<T[], AsyncFree>;
using event_ptr = std::unique_ptr<CUevent_st, EventDestroy>;
using stream_ptr = std::unique_ptr<CUstream_st, StreamDestroy>;
using graph_exec_ptr = std::unique_ptr<CUgraphExec_st, GraphExecDestroy>;
using host_reg_ptr = std::unique_ptr<void, HostUnregister>;

struct tskv_ctx {
  int device = 0;
  stream_ptr stream;
  event_ptr ev0, ev1;
  stream_ptr bin_stream[N_BINS];  // the per-bin fused kernels run concurrently
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

// Tombstone tables (tskvgpu_pages_set_tombstones): the all-series ranges first, then one CSR row per (series, column) key
struct TombTables {
  dev_ptr<uint64_t> keys;
  dev_ptr<uint32_t> off;
  dev_ptr<tskv_time_range> ranges;
  uint32_t n_keys = 0, n_global = 0, n_ranges = 0;
};

// Overlapping chunks (tskvgpu_pages_set_chunk_files, merge_kernels.cuh): the plan, its device copies and the merge rows'
// timestamps (decoded once)
struct OverlapTables {
  OverlapPlan plan;
  dev_ptr<uint8_t> d_cg_merge;
  dev_ptr<int64_t> d_merge_ts;
  dev_ptr<uint64_t> d_mcg_row0, d_mcg_bm0;
  dev_ptr<uint32_t> d_mcg_cg, d_mcg_stream, d_stream_group, d_stream_first_mcg, d_group_first_stream;
  std::vector<uint64_t> h_mcg_bm0;
  uint64_t merge_rows = 0, merge_bm_words = 0;
};

struct tskv_pages {
  tskv_ctx *ctx = nullptr;
  dev_ptr<uint8_t> d_arena;          // device copy (or, host-resident mode: gather target)
  const uint8_t *h_mapped = nullptr; // host-resident mode: device-visible alias of the caller's arena
  bool verify_on_read = false;       // host-resident + VERIFY_CRC: CRC32 checked on the device on every scan
  dev_ptr<uint32_t> d_crc_tables;
  host_reg_ptr h_registered;         // range this library page-locked
  uint64_t arena_len = 0;
  dev_ptr<tskv_page_desc> d_descs;
  std::vector<tskv_page_desc> h_descs;  // with .reserved = DK kind
  uint64_t n_descs = 0;
  dev_ptr<uint32_t> d_time_page_of;
  uint32_t n_cg = 0;
  dev_ptr<uint32_t> d_cg_time_page;
  dev_ptr<uint32_t> d_cg_series_rank;
  dev_ptr<uint32_t> d_series_sorted;  // the page set's distinct series ids, ascending (rank -> id)
  // dense ids (plan_series_map): rank of id series_min + k at d_rank_of[k], k < series_span (null: binary search)
  dev_ptr<uint32_t> d_rank_of;
  uint32_t series_min = 0, series_span = 0;
  dev_ptr<uint32_t> d_rank_cg_start, d_rank_cg;  // CSR: series rank -> its column groups (arena order)
  uint32_t max_series_cg = 0;           // most column groups of one series (plan_walk_split)
  dev_ptr<uint8_t> d_page_bin;          // decode-kind bin of every field page
  mutable dev_ptr<int64_t> d_page_stats;  // {min key, max key} of every field page (k_page_stats), built on first use
  uint32_t n_items = 0;              // field pages
  uint32_t h_bin_pages[N_BINS]{};    // field pages per bin
  // field pages per column id, then per (bin, narrow flag) at bin * WL_SUB + flag: the capacity of a scan's work-list
  // bucket of that column
  std::unordered_map<uint16_t, std::vector<uint32_t>> col_bucket_pages;
  uint64_t h_bin_bytes[N_BINS]{};    // field-page bytes per bin (orders the PCIe gathers of host-resident scans)
  uint64_t h_bin_rows[N_BINS]{};     // rows of the bin's field pages (serial cost of its chunks)
  // the epoch invalidates scans prepared before a change of the tombstones
  TombTables tomb;
  uint64_t tomb_epoch = 0;
  std::vector<uint32_t> series;  // sorted distinct ids
  // arena-wide time bounds, computed on first use by k_time_bounds (the reference keeps them in
  // PageMeta.statistics); only unbucketed first/last across series needs them
  mutable bool bounds_known = false;
  mutable int64_t ts_min = INT64_MIN, ts_max = INT64_MAX;
  // per-column-group [min_ts, max_ts] (ColumnGroup::time_range()): handed in by the caller
  // (tskvgpu_pages_set_time_bounds) or computed together with the arena-wide bounds; drives statistics pruning
  mutable dev_ptr<tskv_time_range> d_cg_bounds;
  // row-filter masks: 32-bit words per column group, offset stored at the index of the group's time page
  dev_ptr<uint32_t> d_keep_off;
  uint64_t keep_words = 0;
  // restart points (skip_kernels.cuh): per page the index of its first entry (or SKIP_NONE), built once at upload
  dev_ptr<uint32_t> d_skip_off;
  dev_ptr<SkipEntry> d_skip;
  uint64_t n_skip = 0;
  // per page 1 = a simple8b integer page whose values all lie in [-2^31, 2^31) (i64) / [0, 2^31) (u64) (k_build_skip;
  // null for host-resident page sets: every page is then wide), and per bin whether none, some or all of its pages are
  // narrow (NARROW_*: which variant of the fused kernel runs the bin)
  dev_ptr<uint8_t> d_narrow;
  uint8_t h_bin_narrow[N_BINS]{};
  uint32_t h_bin_maxrows[N_BINS]{};  // longest field page of each bin (parts per page when a scan cuts the bin's pages)
  std::vector<uint32_t> h_cg_time_page, h_cg_series;
  std::vector<uint8_t> h_time_has_nulls;
  std::vector<tskv_time_range> h_cg_bounds;
  // the epoch invalidates scans prepared before a change of the chunk files
  OverlapTables overlap;
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
  // device buffers, stream-ordered on the context stream (cudaMallocAsync): no device-wide synchronisation on the query
  // path, memory is recycled by the pool
  async_ptr<uint32_t> d_series;
  async_ptr<int32_t> d_rank_slot;  // rank of a series in the page set -> position in the selection list (or -1)
  // selection-driven work list: [N_BINS * n_cols * WL_SUB] fill counts of the buckets, and their regions (+ 1: the end)
  async_ptr<uint32_t> d_bucket, d_region;
  bool split_narrow = false;       // the work list keeps narrow pages in buckets of their own (some bin has both kinds)
  uint32_t walk_split_log2 = 0;    // log2 of the work-list walk's threads per series (plan_walk_split)
  async_ptr<int32_t> d_cg_slot;
  async_ptr<uint32_t> d_work_page, d_work_slot;
  async_ptr<uint8_t> d_work_qcol;
  async_ptr<ColState> d_cols;
  async_ptr<OutCol> d_outs;
  async_ptr<MeanExport> d_means;
  uint32_t n_means = 0;
  async_ptr<uint64_t> d_state;
  async_ptr<unsigned long long> d_aux;  // the aux block (AUX_*); the pointers below point into it
  int32_t *d_status = nullptr;
  unsigned long long *d_err_page = nullptr;
  unsigned long long *d_stats = nullptr;     // [0] points [1] rows in range
  unsigned long long *d_counters = nullptr;  // CTR_*
  async_ptr<uint64_t> d_values;
  async_ptr<uint8_t> d_validity;
  int grid[N_BINS] = {0};
  int occ[N_BINS] = {0};  // resident CTAs per SM of each bin's kernel at this scan's shared memory size
  tskv_ctx *ctx = nullptr;
  uint32_t n_series_sel = 0;
  bool enqueued = false;
  // timing / ordering events of THIS scan (several scans of one context may be in flight from different host threads)
  event_ptr ev0, ev1;
  event_ptr ev_bin[N_BINS + 1];  // [0] fork, [N_BINS] join of the fused phase
  event_ptr ev_bin_start[N_BINS], ev_bin_done[N_BINS], ev_gather[N_BINS];
  tskv_counters counters{};  // of the last completed pass of this scan
  // A scan that is enqueued repeatedly replays its whole pass (2 memsets, ~7 small kernels, the fused kernels forked
  // over the bin streams, export) as ONE CUDA graph launch: captured on the second enqueue, so one-shot scans never pay
  // for a capture.
  graph_exec_ptr graph_exec;
  event_ptr ev_cfork, ev_cjoin[N_BINS];  // dependency-only events of the captured pass
  int32_t *d_crc_status = nullptr;  // a CRC mismatch outranks whatever the decoders made of the bad page
  unsigned long long *d_crc_err_page = nullptr;
  uint32_t n_enqueued = 0;
  bool graph_failed = false;
  PruneRanges prune{};
  async_ptr<uint64_t> d_gathered;  // all ranks' exchange regions (tskvgpu_scan_exchange)
  PredicateSet preds{};            // pushed field predicates (row filter)
  async_ptr<uint32_t> d_row_keep;  // one keep bit per row of every column group (k_row_filter)
  // merge pass over the overlapping chunks this scan reads (merge_kernels.cuh)
  uint64_t chunk_epoch = 0;
  MergeParams merge{};
  uint32_t n_merge_pages = 0;      // field pages decoded per pass
  uint64_t merge_page_bytes = 0, merge_read_pages = 0;
  async_ptr<uint8_t> d_mcg_active;
  async_ptr<uint64_t> d_mvals;
  async_ptr<uint32_t> d_mvalid;
  async_ptr<uint32_t> d_mpage;
  async_ptr<uint64_t> d_mrow_off, d_mbm_off;
  // Layout of the state the fused kernels write at params.state: d_state / sl for a tumbling scan. A sliding scan's
  // kernels fill d_pane_state (panes one slide wide) and k_window_combine folds every run of win_k panes into the
  // windows of d_state / sl, which export, exchange, partials and finalize see.
  StateLayout kern_sl{};
  async_ptr<uint64_t> d_pane_state;
  async_ptr<CombineOp> d_combine;
  uint32_t n_combine = 0, win_k = 1, n_panes = 0, n_windows = 0;
  // GROUP BY tags: the group of every slot (params.slot_group) and the work-list walk order, slots sorted by group (null
  // when that is the selection order)
  async_ptr<uint32_t> d_slot_group, d_walk;
  // explicit time-bucket edges (params.edges; tskvgpu_scan_prepare_edges / _labels), null otherwise; a labelled scan's
  // labels (uint32) follow its n + 1 edges
  async_ptr<int64_t> d_edges;
  // TSKV_AGG_M2 (k_m2_prep, k_scan_m2): its columns, pass 2's parameters and column table, pass 2's bucket fills followed
  // by its task counters, the bins pass 2 runs, the shift / sum(d) / sum(d^2) words at the end of the exchange region
  uint32_t n_m2 = 0;
  async_ptr<M2Col> d_m2;
  async_ptr<ColState> d_cols2;
  async_ptr<uint32_t> d_fill2;
  ScanParams params2{};
  bool m2_bin[N_BINS] = {false};
  uint64_t m2_words = 0;
  event_ptr ev_m2_fork, ev_m2_join[N_BINS];
  // column pairs (tskv_query.n_pairs; k_scan_pair): their state sections, which follow the M2 ones in the exchange region
  uint32_t n_pairs = 0;
  async_ptr<PairCol> d_pairs;
  uint64_t pair_words = 0;
  // medians (TSKV_QUERY_N_MEDIANS; k_scan_median): their operands, selection state (MedianSec sections, then the count of
  // unresolved cells) and histograms
  uint32_t n_medians = 0;
  async_ptr<MedianCol> d_medians;
  async_ptr<uint64_t> d_med_state;
  async_ptr<uint32_t> d_med_hist;
  MedianArgs med{};
  // increases (TSKV_QUERY_N_INCREASES; k_scan_increase): their operands, records (IncreaseArgs: n_rec per increase, the
  // operand's work items then the merge rows), the sorts' key and index buffers and scratch
  uint32_t n_increases = 0;
  uint64_t n_inc_merge_rows = 0;
  int inc_time_sort_bits = 64, inc_slot_sort_bits = 64;  // the key bits each sort reads
  async_ptr<IncreaseCol> d_increases;
  async_ptr<uint32_t> d_inc_rec0;      // IncreaseArgs::rec0
  async_ptr<ulonglong4> d_inc_rec;
  async_ptr<uint64_t> d_inc_keys;  // slot keys, time keys, sorted time keys, slot keys in time order, sorted slot keys
  async_ptr<uint32_t> d_inc_idx;   // identity, after the time sort, after the slot sort
  async_ptr<uint8_t> d_inc_tmp;
  size_t inc_tmp_bytes = 0;
  IncreaseArgs inc{};
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

// Fill `p` with n elements; a zero-length array still gets one element (a valid, distinct address).
template <typename T>
cudaError_t dev_alloc(dev_ptr<T> &p, size_t n) {
  T *raw = nullptr;
  const cudaError_t e = cudaMalloc(reinterpret_cast<void **>(&raw), std::max<size_t>(n, 1) * sizeof(T));
  p.reset(e == cudaSuccess ? raw : nullptr);
  return e;
}
// Stream-ordered on `stream`, and freed on it.
template <typename T>
cudaError_t stream_alloc(async_ptr<T> &p, size_t n, cudaStream_t stream) {
  T *raw = nullptr;
  const cudaError_t e = cudaMallocAsync(reinterpret_cast<void **>(&raw), std::max<size_t>(n, 1) * sizeof(T), stream);
  p = async_ptr<T>(e == cudaSuccess ? raw : nullptr, AsyncFree{stream});
  return e;
}
// Allocates n elements as dev_alloc / stream_alloc do and copies src[0, n) into them on `stream`. The copy is ordered
// before any later work on `stream`; src must stay alive until then or until the stream is synchronised.
template <typename T, typename Free>
cudaError_t upload(std::unique_ptr<T[], Free> &p, const T *src, size_t n, cudaStream_t stream) {
  cudaError_t e;
  if constexpr (std::is_same_v<Free, AsyncFree>) e = stream_alloc(p, n, stream);
  else e = dev_alloc(p, n);
  if (e == cudaSuccess && n) e = cudaMemcpyAsync(p.get(), src, n * sizeof(T), cudaMemcpyHostToDevice, stream);
  return e;
}
// Copies src[0, n) into a page set's table on `stream` and waits for the copy. A table already in place is overwritten
// where it lies: a scan captured into a CUDA graph holds its address. A new table is published only once it is filled.
template <typename T>
cudaError_t fill_table(dev_ptr<T> &table, const T *src, size_t n, cudaStream_t stream) {
  dev_ptr<T> fresh;
  cudaError_t e = table ? cudaSuccess : dev_alloc(fresh, n);
  if (e == cudaSuccess && n) e = cudaMemcpyAsync(table ? table.get() : fresh.get(), src, n * sizeof(T), cudaMemcpyHostToDevice, stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(stream);
  if (e == cudaSuccess && fresh) table = std::move(fresh);
  return e;
}

event_ptr new_event(unsigned flags = cudaEventDefault) {
  cudaEvent_t ev = nullptr;
  return event_ptr(cudaEventCreateWithFlags(&ev, flags) == cudaSuccess ? ev : nullptr);
}

unsigned bits_for(uint64_t max_value) {  // bits needed to represent values in [0, max_value]
  unsigned b = 0;
  while (max_value) {
    b++;
    max_value >>= 1;
  }
  return b;
}

unsigned popc8(unsigned x) { return (unsigned)__builtin_popcount(x & 0xffu); }

// The aggregates the pass-1 kernels compute for a column: its own, and for TSKV_AGG_M2 also the COUNT and the exact SUM
// that MEAN keeps (pass 2 shifts by that mean). The M2 bit itself never reaches them.
uint8_t kernel_mask(uint8_t m) { return (uint8_t)((m & TSKV_AGG_ALL) | ((m & TSKV_AGG_M2) ? TSKV_AGG_MEAN : 0)); }

bool query_has_m2(const tskv_query *q) {
  for (uint32_t c = 0; c < q->n_columns; c++)
    if (q->columns[c].agg_mask & TSKV_AGG_M2) return true;
  return false;
}

uint32_t query_n_medians(const tskv_query *q) { return TSKV_QUERY_N_MEDIANS(q->reserved); }
uint32_t query_n_increases(const tskv_query *q) { return TSKV_QUERY_N_INCREASES(q->reserved); }

// The query the scan runs for a query with column pairs, medians or increases: its projected columns, then every operand that is
// not one of them as a COUNT column without output (so that the work list, the page gathers, CRC checks, pass 1 and the
// reader counters treat the operands' pages as they treat a COUNT column's), and per pair, median and increase the
// operands' places in that table. A median's operand column also computes MIN and MAX in pass 1 (its extreme keys); an increase's
// operand column computes COUNT (its validity).
struct OperandQuery {
  tskv_query q{};
  std::vector<tskv_agg_column> cols;
  std::vector<PairCol> pairs;          // (off is set by plan_layout)
  std::vector<MedianCol> medians;      // (the offsets are set by plan_layout)
  std::vector<IncreaseCol> increases;  // (the offsets are set by plan_layout)
};
OperandQuery plan_operand_query(const tskv_query *q) {
  OperandQuery pq;
  pq.q = *q;
  pq.cols.assign(q->columns, q->columns + q->n_columns);
  auto place = [&](const tskv_agg_column &op) {
    for (uint32_t c = 0; c < pq.cols.size(); c++)
      if (pq.cols[c].column_id == op.column_id) return c;
    pq.cols.push_back(tskv_agg_column{op.column_id, op.phys_type, (uint8_t)TSKV_AGG_COUNT});
    return (uint32_t)pq.cols.size() - 1;
  };
  for (uint32_t p = 0; p < q->n_pairs; p++) {
    const tskv_agg_column &x = q->columns[q->n_columns + 2 * p], &y = q->columns[q->n_columns + 2 * p + 1];
    PairCol pc{};
    pc.qx = place(x);
    pc.qy = place(y);
    pc.x_id = x.column_id;
    pc.y_id = y.column_id;
    pc.x_pt = x.phys_type;
    pc.y_pt = y.phys_type;
    pq.pairs.push_back(pc);
  }
  for (uint32_t m = 0; m < query_n_medians(q); m++) {
    const tskv_agg_column &op = q->columns[q->n_columns + 2 * q->n_pairs + m];
    MedianCol mc{};
    mc.qcol = place(op);
    pq.cols[mc.qcol].agg_mask |= TSKV_AGG_MIN | TSKV_AGG_MAX;
    mc.column_id = op.column_id;
    mc.phys_type = op.phys_type;
    pq.medians.push_back(mc);
  }
  for (uint32_t k = 0; k < query_n_increases(q); k++) {
    const tskv_agg_column &op = q->columns[q->n_columns + 2 * q->n_pairs + query_n_medians(q) + k];
    IncreaseCol ic{};
    ic.qcol = place(op);
    pq.cols[ic.qcol].agg_mask |= TSKV_AGG_COUNT;
    ic.column_id = op.column_id;
    ic.phys_type = op.phys_type;
    pq.increases.push_back(ic);
  }
  pq.q.columns = pq.cols.data();
  pq.q.n_columns = (uint32_t)pq.cols.size();
  return pq;
}

typedef void (*scan_kernel_t)(const ScanParams, int);
// `narrow`: NARROW_* of the bin's pages (tskv_pages::h_bin_narrow); only the simple8b-value kernels without FIRST / LAST
// have narrow variants; EDGES: the kernels of an edge scan (ScanParams.edges)
template <bool SEL, bool EDGES>
scan_kernel_t scan_kernel_for(int bin, int narrow = NARROW_NONE) {
  if constexpr (!SEL) {
    if (narrow == NARROW_SOME && bin == TK_RLE * N_VK + VK_S8B) return k_scan_aggregate<TK_RLE, VK_S8B, false, NARROW_SOME, EDGES>;
    if (narrow == NARROW_SOME && bin == TK_S8B * N_VK + VK_S8B) return k_scan_aggregate<TK_S8B, VK_S8B, false, NARROW_SOME, EDGES>;
    if (narrow == NARROW_ALL && bin == TK_RLE * N_VK + VK_S8B) return k_scan_aggregate<TK_RLE, VK_S8B, false, NARROW_ALL, EDGES>;
    if (narrow == NARROW_ALL && bin == TK_S8B * N_VK + VK_S8B) return k_scan_aggregate<TK_S8B, VK_S8B, false, NARROW_ALL, EDGES>;
  }
  switch (bin) {
    case TK_RLE * N_VK + VK_S8B: return k_scan_aggregate<TK_RLE, VK_S8B, SEL, NARROW_NONE, EDGES>;
    case TK_RLE * N_VK + VK_GOR: return k_scan_aggregate<TK_RLE, VK_GOR, SEL, NARROW_NONE, EDGES>;
    case TK_RLE * N_VK + VK_GEN: return k_scan_aggregate<TK_RLE, VK_GEN, SEL, NARROW_NONE, EDGES>;
    case TK_S8B * N_VK + VK_S8B: return k_scan_aggregate<TK_S8B, VK_S8B, SEL, NARROW_NONE, EDGES>;
    case TK_S8B * N_VK + VK_GOR: return k_scan_aggregate<TK_S8B, VK_GOR, SEL, NARROW_NONE, EDGES>;
    case TK_S8B * N_VK + VK_GEN: return k_scan_aggregate<TK_S8B, VK_GEN, SEL, NARROW_NONE, EDGES>;
    case TK_GEN * N_VK + VK_S8B: return k_scan_aggregate<TK_GEN, VK_S8B, SEL, NARROW_NONE, EDGES>;
    case TK_GEN * N_VK + VK_GOR: return k_scan_aggregate<TK_GEN, VK_GOR, SEL, NARROW_NONE, EDGES>;
    default: return k_scan_aggregate<TK_GEN, VK_GEN, SEL, NARROW_NONE, EDGES>;
  }
}
template <bool SEL>
scan_kernel_t scan_kernel_for(int bin, bool edges, int narrow = NARROW_NONE) {
  return edges ? scan_kernel_for<SEL, true>(bin, narrow) : scan_kernel_for<SEL, false>(bin, narrow);
}
// pass 2 of TSKV_AGG_M2 (k_scan_m2): one kernel per serial bin (narrow pages take the wide arithmetic)
template <bool EDGES>
scan_kernel_t m2_kernel_for(int bin) {
  switch (bin) {
    case TK_RLE * N_VK + VK_S8B: return k_scan_m2<TK_RLE, VK_S8B, EDGES>;
    case TK_RLE * N_VK + VK_GOR: return k_scan_m2<TK_RLE, VK_GOR, EDGES>;
    case TK_RLE * N_VK + VK_GEN: return k_scan_m2<TK_RLE, VK_GEN, EDGES>;
    case TK_S8B * N_VK + VK_S8B: return k_scan_m2<TK_S8B, VK_S8B, EDGES>;
    case TK_S8B * N_VK + VK_GOR: return k_scan_m2<TK_S8B, VK_GOR, EDGES>;
    case TK_S8B * N_VK + VK_GEN: return k_scan_m2<TK_S8B, VK_GEN, EDGES>;
    case TK_GEN * N_VK + VK_S8B: return k_scan_m2<TK_GEN, VK_S8B, EDGES>;
    case TK_GEN * N_VK + VK_GOR: return k_scan_m2<TK_GEN, VK_GOR, EDGES>;
    default: return k_scan_m2<TK_GEN, VK_GEN, EDGES>;
  }
}
scan_kernel_t m2_kernel_for(int bin, bool edges) { return edges ? m2_kernel_for<true>(bin) : m2_kernel_for<false>(bin); }
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
  dev_ptr<long long> d_bounds;
  if (dev_alloc(d_bounds, 2) != cudaSuccess) return;
  long long b[2] = {INT64_MAX, INT64_MIN};
  cudaMemcpyAsync(d_bounds.get(), b, sizeof(b), cudaMemcpyHostToDevice, ctx->stream.get());
  if (!pg->d_cg_bounds) dev_alloc(pg->d_cg_bounds, pg->n_cg);
  k_time_bounds<<<(pg->n_cg + 127) / 128, 128, 0, ctx->stream.get()>>>(pg->h_mapped ? pg->h_mapped : pg->d_arena.get(), pg->d_descs.get(),
                                                                pg->d_cg_time_page.get(), pg->n_cg, d_bounds.get(), pg->d_cg_bounds.get());
  if (cudaMemcpyAsync(b, d_bounds.get(), sizeof(b), cudaMemcpyDeviceToHost, ctx->stream.get()) == cudaSuccess &&
      cudaStreamSynchronize(ctx->stream.get()) == cudaSuccess && b[0] <= b[1]) {
    pg->ts_min = b[0];
    pg->ts_max = b[1];
  }
  pg->bounds_known = true;
}

// Value statistics of the field pages, computed on the device the first time a scan with field predicates is prepared
// (pages resident in HBM only; the reference reads them from PageMeta.statistics).
void ensure_page_stats(tskv_ctx *ctx, const tskv_pages *pg) {
  static const bool off = getenv("TSKV_NO_VALUE_STATS") != nullptr;
  if (off || pg->d_page_stats || pg->h_mapped || pg->n_descs == 0) return;
  dev_ptr<int64_t> d;
  if (dev_alloc(d, 2 * (size_t)pg->n_descs) != cudaSuccess) {
    cudaGetLastError();
    return;
  }
  k_page_stats<<<(unsigned)((pg->n_descs + 127) / 128), 128, 0, ctx->stream.get()>>>(pg->d_arena.get(), pg->d_descs.get(), pg->n_descs, d.get());
  if (cudaGetLastError() != cudaSuccess || cudaStreamSynchronize(ctx->stream.get()) != cudaSuccess) return;
  pg->d_page_stats = std::move(d);
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

// Explicit time-bucket edges (the *_edges and *_labels entry points; `on`): n edge buckets [edges[b], edges[b + 1]).
// labelled (the *_labels calls): edge bucket b aggregates into output bucket labels[b] < q->n_buckets. Otherwise the edge
// buckets are the output buckets, n = q->n_buckets.
struct BucketEdges {
  bool on = false;
  const int64_t *edges = nullptr;
  uint32_t n = 0;
  bool labelled = false;
  const uint32_t *labels = nullptr;
};

// Why an explicit time-bucket edge table or its labels are refused (TSKV_ERR_INVALID_ARG), or null.
const char *edges_refusal(const tskv_query *q, const BucketEdges &E) {
  if (!E.on) return nullptr;
  if (E.labelled) {
    if (!E.labels || E.n == 0 || q->n_buckets == 0)
      return "bucket labels: labels must be non-null, n_edge >= 1 and n_buckets >= 1";
    for (uint32_t b = 0; b < E.n; b++)
      if (E.labels[b] >= q->n_buckets) return "bucket labels: a label is >= n_buckets";
  }
  if (!E.edges || E.n == 0) return "time-bucket edges: edges must be non-null and n_buckets >= 1";
  if (q->width != 0 || q->origin != 0 || q->first_bucket_start != 0)
    return "time-bucket edges: width, origin and first_bucket_start must be 0 (the edges replace them)";
  for (uint32_t b = 0; b < E.n; b++)
    if (E.edges[b + 1] <= E.edges[b]) return "time-bucket edges: the edges must be strictly increasing";
  if ((uint64_t)E.edges[E.n] - (uint64_t)E.edges[0] >= 1ull << 63)
    return "time-bucket edges: edges[n_buckets] - edges[0] must be below 2^63";
  return nullptr;
}

// Labelled edge scans refuse FIRST / LAST (TSKV_ERR_UNSUPPORTED): the reference takes a record batch's earliest row per
// label, and the NULL rule at that row then acts across the page's edge buckets of one label (DESIGN.md section 7).
bool labels_first_last(const tskv_query *q, const BucketEdges &E) {
  if (!E.labelled) return false;
  for (uint32_t c = 0; c < q->n_columns; c++)
    if (q->columns[c].agg_mask & (TSKV_AGG_FIRST | TSKV_AGG_LAST)) return true;
  return false;
}

// (an edge scan's buckets come from its edge table, width = 0)
bool query_shape_ok(const tskv_query *q, bool edges = false) {
  return q->n_buckets != 0 &&
         (q->n_columns != 0 || q->n_pairs != 0 || query_n_medians(q) != 0 || query_n_increases(q) != 0) && q->columns &&
         (q->width > 0 || q->n_buckets == 1 || edges);
}

// Output layout of a query that passed query_shape_ok and tag_groups_refusal.
tskv_output_layout output_layout(const tskv_pages *pages, const tskv_query *q, const TagGroups &tg) {
  tskv_output_layout out;
  uint64_t n_out = 0;
  for (uint32_t c = 0; c < q->n_columns; c++) n_out += popc8(q->columns[c].agg_mask);
  if (q->n_pairs <= TSKV_MAX_PAIRS) n_out += 4ull * q->n_pairs;  // n, C, M2x, M2y per pair
  if (query_n_medians(q) <= TSKV_MAX_MEDIANS) n_out += query_n_medians(q);
  if (query_n_increases(q) <= TSKV_MAX_INCREASES) n_out += query_n_increases(q);
  uint64_t n_groups = 1;
  if (q->group_by_series) n_groups = selected_slots(pages, q);
  if (tg.on) n_groups = tg.n;
  out.n_out = n_out;
  out.n_groups = n_groups;
  out.n_cells = n_groups * q->n_buckets;
  out.bitmap_stride = (out.n_cells + 63) / 64 * 8;
  out.values_bytes = n_out * out.n_cells * 8;
  out.validity_bytes = n_out * out.bitmap_stride;
  return out;
}

// E.on: an edge scan's layout (tskvgpu_query_output_layout_edges / _labels), with its refusals.
tskv_status compute_layout(const tskv_pages *pages, const tskv_query *q, const TagGroups &tg, const BucketEdges &E,
                           tskv_output_layout *out) {
  if (!pages || !q || !out || edges_refusal(q, E) || !query_shape_ok(q, E.on) || tag_groups_refusal(pages, q, tg))
    return TSKV_ERR_INVALID_ARG;
  if (labels_first_last(q, E)) return TSKV_ERR_UNSUPPORTED;
  *out = output_layout(pages, q, tg);
  return TSKV_OK;
}

// Offsets of the partial state of `q` over n_cells cells: the sections tskv_partials_view exposes, in that order, then
// the scan's own arrays (first / last pairs, key snapshot, high words of exact integer sums).
struct StatePlan {
  StateLayout sl{};
  std::vector<ColState> cols;
  std::vector<MeanExport> means;
  std::vector<uint64_t> msum_off;  // per column: the exported f64 exact integer sum of MEAN, or 0
  std::vector<M2Col> m2;           // TSKV_AGG_M2 columns, in query order
  std::vector<int> m2_of;          // per column: its index in m2, or -1
  uint64_t m2_words = 0;           // their shift / sum(d) / sum(d^2) sections, which follow the values section
  uint64_t pair_off = 0, pair_words = 0;  // the column pairs' sections (PAIR_WORDS per pair), after the M2 ones
  std::vector<uint64_t> inc_off;          // per increase: its sum section, after the integer / the f64 sums
};
// incs: the increases (plan_operand_query's), whose sums the exchange region's sum sections hold
StatePlan plan_state(const tskv_query *q, uint64_t n_cells, const std::vector<IncreaseCol> &incs = {}) {
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
    cols[c].agg_mask = kernel_mask(qc.agg_mask);
    cols[c].count_off = off;
    off += n_cells;
    if ((kernel_mask(qc.agg_mask) & (TSKV_AGG_SUM | TSKV_AGG_MEAN)) && qc.phys_type != TSKV_PT_F64) {
      cols[c].sum_off = off;
      off += n_cells;
    }
  }
  plan.inc_off.assign(incs.size(), 0);
  for (size_t k = 0; k < incs.size(); k++)
    if (incs[k].phys_type != TSKV_PT_F64) {
      plan.inc_off[k] = off;
      off += n_cells;
    }
  sl.sum_i64_len = off - sl.sum_i64_off;
  sl.sum_f64_off = off;
  for (uint32_t c = 0; c < q->n_columns; c++)
    if ((kernel_mask(q->columns[c].agg_mask) & (TSKV_AGG_SUM | TSKV_AGG_MEAN)) && q->columns[c].phys_type == TSKV_PT_F64) {
      cols[c].sum_off = off;
      off += n_cells;
    }
  for (uint32_t c = 0; c < q->n_columns; c++)
    if ((kernel_mask(q->columns[c].agg_mask) & TSKV_AGG_MEAN) && q->columns[c].phys_type != TSKV_PT_F64) {
      msum_off[c] = off;  // exported exact integer sum as f64 (all-reducible)
      off += n_cells;
    }
  for (size_t k = 0; k < incs.size(); k++)
    if (incs[k].phys_type == TSKV_PT_F64) {
      plan.inc_off[k] = off;
      off += n_cells;
    }
  sl.sum_f64_len = off - sl.sum_f64_off;
  uint64_t n_first = 0, n_last = 0;
  for (uint32_t c = 0; c < q->n_columns; c++) {
    if (kernel_mask(q->columns[c].agg_mask) & TSKV_AGG_FIRST) n_first += n_cells;
    if (kernel_mask(q->columns[c].agg_mask) & TSKV_AGG_LAST) n_last += n_cells;
  }
  sl.first_cells = n_first;
  sl.last_cells = n_last;
  sl.min_off = off;
  for (uint32_t c = 0; c < q->n_columns; c++)
    if (kernel_mask(q->columns[c].agg_mask) & TSKV_AGG_MIN) {
      cols[c].min_off = off;
      off += n_cells;
    }
  sl.first_keys_off = off;
  off += n_first;
  sl.min_len = off - sl.min_off;
  sl.max_off = off;
  for (uint32_t c = 0; c < q->n_columns; c++)
    if (kernel_mask(q->columns[c].agg_mask) & TSKV_AGG_MAX) {
      cols[c].max_off = off;
      off += n_cells;
    }
  sl.last_keys_off = off;
  off += n_last;
  sl.max_len = off - sl.max_off;
  sl.selval_off = off;
  off += n_first + n_last;
  sl.selval_len = n_first + n_last;
  // TSKV_AGG_M2: the cells' shifts, sum(d) and sum(d^2), right after the values so that the exchange region holds them
  plan.m2_of.assign(q->n_columns, -1);
  for (uint32_t c = 0; c < q->n_columns; c++)
    if (q->columns[c].agg_mask & TSKV_AGG_M2) {
      plan.m2_of[c] = (int)plan.m2.size();
      plan.m2.push_back(M2Col{cols[c].count_off, msum_off[c] ? msum_off[c] : cols[c].sum_off, off, off + n_cells, off + 2 * n_cells});
      off += 3 * n_cells;
    }
  plan.m2_words = 3 * n_cells * plan.m2.size();
  plan.pair_off = off;
  plan.pair_words = (uint64_t)PAIR_WORDS * n_cells * q->n_pairs;
  off += plan.pair_words;
  off = (off + 1) & ~1ull;  // 16-byte alignment of the pair arrays
  sl.first_pairs_off = off;
  {
    uint64_t o = off;
    for (uint32_t c = 0; c < q->n_columns; c++)
      if (kernel_mask(q->columns[c].agg_mask) & TSKV_AGG_FIRST) {
        cols[c].first_off = o;
        o += 2 * n_cells;
      }
    off = o;
  }
  sl.last_pairs_off = off;
  {
    uint64_t o = off;
    for (uint32_t c = 0; c < q->n_columns; c++)
      if (kernel_mask(q->columns[c].agg_mask) & TSKV_AGG_LAST) {
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

// Reads back the device status word; maps it to a message.
tskv_status fetch_status(tskv_ctx *ctx, int32_t *d_status, unsigned long long *d_err_page) {
  int32_t st = 0;
  unsigned long long pg = 0;
  if (cudaMemcpyAsync(&st, d_status, sizeof(st), cudaMemcpyDeviceToHost, ctx->stream.get()) != cudaSuccess ||
      cudaMemcpyAsync(&pg, d_err_page, sizeof(pg), cudaMemcpyDeviceToHost, ctx->stream.get()) != cudaSuccess ||
      cudaStreamSynchronize(ctx->stream.get()) != cudaSuccess) {
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

// Narrows [lo, hi] to the span of the query's time ranges (no ranges: every timestamp); lo > hi: nothing in range.
void clip_to_query_ranges(const tskv_query *q, int64_t &lo, int64_t &hi) {
  if (q->n_time_ranges == 0) return;
  int64_t qlo = q->time_ranges[0].min_ts, qhi = q->time_ranges[0].max_ts;
  for (uint32_t r = 1; r < q->n_time_ranges; r++) {
    qlo = std::min(qlo, q->time_ranges[r].min_ts);
    qhi = std::max(qhi, q->time_ranges[r].max_ts);
  }
  lo = std::max(lo, qlo);
  hi = std::min(hi, qhi);
}

// Sliding windows of `q` (window q->width, slide < q->width) by panes: the refusals of tskvgpu_scan_prepare_sliding
// (DESIGN.md section 7) and the pane grid. Called under ctx->mu.
tskv_status check_sliding(tskv_ctx *ctx, const tskv_pages *pages, const tskv_query *q, int64_t slide, uint32_t *out_k) {
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
    clip_to_query_ranges(q, lo, hi);
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

// The refusals of the tskvgpu_scan_prepare* calls: sets the error and returns its status, or returns TSKV_OK with the
// windows per row (1 unless slide > 0). Called under ctx->mu.
tskv_status validate_query(tskv_ctx *ctx, const tskv_pages *pages, const tskv_query *q, int64_t slide, const TagGroups &tg,
                           const BucketEdges &E, uint32_t *win_k) {
  if (const char *why = edges_refusal(q, E)) {  // the *_edges and *_labels calls
    ctx->set_error(why);
    return TSKV_ERR_INVALID_ARG;
  }
  if (const char *why = tag_groups_refusal(pages, q, tg)) {
    ctx->set_error(why);
    return TSKV_ERR_INVALID_ARG;
  }
  if (!query_shape_ok(q, E.on)) {
    ctx->set_error("invalid query (buckets / columns)");
    return TSKV_ERR_INVALID_ARG;
  }
  if (q->n_columns > 126 || q->n_time_ranges > MAX_RANGES || (q->n_time_ranges && !q->time_ranges)) {
    ctx->set_error("invalid query: at most 126 columns and 8 time ranges");
    return TSKV_ERR_INVALID_ARG;
  }
  if (q->n_pairs > TSKV_MAX_PAIRS || (uint64_t)q->n_columns + 2ull * q->n_pairs > 126) {
    ctx->set_error("invalid query: at most 8 column pairs and 126 columns with the pairs' operands");
    return TSKV_ERR_INVALID_ARG;
  }
  for (uint32_t k = 0; k < 2 * q->n_pairs; k++) {
    const tskv_agg_column &op = q->columns[q->n_columns + k];
    if (op.agg_mask != 0 || op.phys_type < TSKV_PT_I64 || op.phys_type > TSKV_PT_F64) {
      ctx->set_error("invalid pair operand: an I64 / U64 / F64 column with agg_mask 0");
      return TSKV_ERR_INVALID_ARG;
    }
    for (uint32_t c = 0; c < q->n_columns + k; c++)
      if (q->columns[c].column_id == op.column_id && q->columns[c].phys_type != op.phys_type) {
        ctx->set_error("pair operand: one column id with two types");
        return TSKV_ERR_INVALID_ARG;
      }
  }
  const uint32_t n_med = query_n_medians(q);
  if (n_med > TSKV_MAX_MEDIANS || (uint64_t)q->n_columns + 2ull * q->n_pairs + n_med > 126) {
    ctx->set_error("invalid query: at most 8 medians and 126 columns with the pairs' and medians' operands");
    return TSKV_ERR_INVALID_ARG;
  }
  for (uint32_t k = 2 * q->n_pairs; k < 2 * q->n_pairs + n_med; k++) {
    const tskv_agg_column &op = q->columns[q->n_columns + k];
    if (op.agg_mask != 0 || op.phys_type < TSKV_PT_I64 || op.phys_type > TSKV_PT_F64) {
      ctx->set_error("invalid median operand: an I64 / U64 / F64 column with agg_mask 0");
      return TSKV_ERR_INVALID_ARG;
    }
    for (uint32_t c = 0; c < q->n_columns + k; c++)
      if (q->columns[c].column_id == op.column_id && q->columns[c].phys_type != op.phys_type) {
        ctx->set_error("median operand: one column id with two types");
        return TSKV_ERR_INVALID_ARG;
      }
  }
  const uint32_t n_inc = query_n_increases(q);
  if (n_inc > TSKV_MAX_INCREASES || (uint64_t)q->n_columns + 2ull * q->n_pairs + n_med + n_inc > 126) {
    ctx->set_error("invalid query: at most 8 increases and 126 columns with the pairs', medians' and increases' operands");
    return TSKV_ERR_INVALID_ARG;
  }
  for (uint32_t k = 2 * q->n_pairs + n_med; k < 2 * q->n_pairs + n_med + n_inc; k++) {
    const tskv_agg_column &op = q->columns[q->n_columns + k];
    if (op.agg_mask != 0 || op.phys_type < TSKV_PT_I64 || op.phys_type > TSKV_PT_F64) {
      ctx->set_error("invalid increase operand: an I64 / U64 / F64 column with agg_mask 0");
      return TSKV_ERR_INVALID_ARG;
    }
    for (uint32_t c = 0; c < q->n_columns + k; c++)
      if (q->columns[c].column_id == op.column_id && q->columns[c].phys_type != op.phys_type) {
        ctx->set_error("increase operand: one column id with two types");
        return TSKV_ERR_INVALID_ARG;
      }
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
    if (qc.phys_type < TSKV_PT_I64 || qc.phys_type > TSKV_PT_BOOL || (qc.agg_mask & ~(TSKV_AGG_ALL | TSKV_AGG_M2)) || qc.agg_mask == 0) {
      ctx->set_error("invalid query column (type or aggregate mask)");
      return TSKV_ERR_INVALID_ARG;
    }
    if (qc.phys_type == TSKV_PT_BOOL && (qc.agg_mask & (TSKV_AGG_SUM | TSKV_AGG_MEAN | TSKV_AGG_M2))) {
      ctx->set_error("sum / mean / m2 of a boolean column");
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
  if (labels_first_last(q, E)) {
    ctx->set_error("bucket labels: first / last are not supported (the reference takes each batch's earliest row per label)");
    return TSKV_ERR_UNSUPPORTED;
  }
  if (slide && query_has_m2(q)) {
    ctx->set_error("sliding windows: M2 (variance) is not pushed down: folding panes would need a Chan merge of their second moments");
    return TSKV_ERR_UNSUPPORTED;
  }
  if (slide && q->n_pairs) {
    ctx->set_error("sliding windows: column pairs (covariance / correlation) are not pushed down");
    return TSKV_ERR_UNSUPPORTED;
  }
  if (n_med && slide) {
    ctx->set_error("sliding windows: medians are not pushed down");
    return TSKV_ERR_UNSUPPORTED;
  }
  if (n_med && (q->reserved & TSKV_QUERY_MULTI_RANK)) {
    ctx->set_error("multi-rank scan: medians are not pushed down (their selection state does not merge across ranks)");
    return TSKV_ERR_UNSUPPORTED;
  }
  if (n_inc) {  // increases pair consecutive rows of one series: a cell must never hold two selected series
    const char *why = nullptr;
    if (slide) why = "sliding windows: increases are not pushed down";
    else if (E.labelled) why = "bucket labels: increases are not pushed down (date_part cells are not monotone in time)";
    else if (tg.on) {
      std::vector<uint8_t> seen(tg.n, 0);
      const uint64_t n_slots = selected_slots(pages, q);
      for (uint64_t i = 0; i < n_slots && !why; i++)
        if (seen[tg.ids[i]]++) why = "increase: a tag group holds two selected series (a cell must hold one series)";
    } else if (!q->group_by_series) {
      // (a multi-rank scan decides from the query alone, so that every rank agrees: without series_ids each rank would
      // count only its own series, and the exchange would sum several series' increases into one cell)
      if (q->series_ids ? q->n_series > 1 : (q->reserved & TSKV_QUERY_MULTI_RANK) || pages->series.size() > 1)
        why = "increase: an ungrouped scan over more than one selected series, or a multi-rank one without series_ids "
              "(a cell must hold one series)";
    }
    if (why) {
      ctx->set_error(why);
      return TSKV_ERR_UNSUPPORTED;
    }
  }
  for (uint32_t m = 0; m < n_med; m++) {  // the histograms count a cell's keys in 32 bits
    const uint16_t id = q->columns[q->n_columns + 2 * q->n_pairs + m].column_id;
    uint64_t rows = 0;
    for (const tskv_page_desc &d : pages->h_descs)
      if (d.phys_type != TSKV_PT_TIME && d.column_id == id) rows += d.num_values;
    if (rows >> 32) {
      ctx->set_error("median: the operand's pages hold 2^32 rows or more");
      return TSKV_ERR_UNSUPPORTED;
    }
  }
  *win_k = 1;
  return slide ? check_sliding(ctx, pages, q, slide, win_k) : TSKV_OK;
}

// FIRST / LAST tie-break key (ScanParams::slot_bits / rel_base) of a scan with FIRST / LAST (has_sel). Refuses
// (TSKV_ERR_UNSUPPORTED) a scan whose keys do not fit 62 bits.
tskv_status plan_keys(tskv_ctx *ctx, const tskv_pages *pages, const tskv_query *q, const BucketEdges &E, bool has_sel,
                      uint32_t *slot_bits, int64_t *rel_base) {
  const uint64_t n_slots = selected_slots(pages, q);
  *slot_bits = (q->group_by_series || n_slots <= 1) ? 0 : bits_for(n_slots - 1);
  *rel_base = 0;
  if (!has_sel || *slot_bits == 0) return TSKV_OK;
  unsigned rel_bits = 64;
  if (E.on) {  // rel = t - edges[b] + 1 in [1, longest bucket]
    uint64_t longest = 0;
    for (uint32_t b = 0; b < E.n; b++) longest = std::max(longest, (uint64_t)E.edges[b + 1] - (uint64_t)E.edges[b]);
    rel_bits = bits_for(longest);
  } else if (q->width > 0) {
    if (q->width < (int64_t)1 << 61) rel_bits = bits_for(2 * (uint64_t)q->width);
  } else {
    // unbucketed: rel = t - (lower bound of every in-range timestamp). A single-rank scan tightens unbounded / loose
    // query ranges with the arena's own time bounds; a scan whose partials are merged with other ranks'
    // (TSKV_QUERY_MULTI_RANK) must build keys every rank agrees on, i.e. from the query alone.
    int64_t lo = INT64_MIN, hi = INT64_MAX;
    if (!(q->reserved & TSKV_QUERY_MULTI_RANK)) {
      ensure_time_bounds(ctx, pages);
      lo = pages->ts_min;
      hi = pages->ts_max;
    }
    clip_to_query_ranges(q, lo, hi);
    if (hi < lo) {
      rel_bits = 0;  // nothing can be in range
    } else {
      rel_bits = bits_for((uint64_t)hi - (uint64_t)lo);
      *rel_base = lo;
    }
  }
  if (rel_bits + *slot_bits > 62) {
    ctx->set_error("first/last across series: (bucket width, longest bucket or time span) x series count does not fit the 62-bit "
                   "tie-break key");
    return TSKV_ERR_UNSUPPORTED;
  }
  return TSKV_OK;
}

// The state of a scan and the tables the host builds from its layout.
struct ScanLayout {
  StateLayout sl{};       // the state export, exchange, partials and finalize see
  StateLayout kern_sl{};  // the state the fused kernels write: sl, or for a sliding scan the panes' state
  std::vector<ColState> cols;      // the fused kernels' column table (offsets into kern_sl's state)
  std::vector<CombineOp> combine;  // a sliding scan: pane state -> window state
  std::vector<MeanExport> means;
  std::vector<OutCol> outs;
  uint32_t use_smem = 0, smem_words = 0;  // the per-CTA shared-memory partial table (ScanParams)
  // TSKV_AGG_M2: its columns, pass 2's column table (k_scan_m2) and shared-memory table, and the shift / sum(d) /
  // sum(d^2) words that extend the exchange region
  std::vector<M2Col> m2;
  std::vector<ColState> cols2;
  uint32_t use_smem2 = 0, smem_words2 = 0;
  uint64_t m2_words = 0;
  std::vector<PairCol> pairs;  // column pairs, with their state offsets
  uint64_t pair_words = 0;
  std::vector<MedianCol> medians;  // medians, with their operands' pass-1 sections and their selection state's offsets
  std::vector<IncreaseCol> increases;  // increases, with their operands' COUNT sections and their sum sections
};

// n_cells: cells of the query's grid (a sliding scan: windows); kern_cells: cells of the fused kernels' grid (panes).
// user_cols[0, n_user): the columns with outputs, as the caller asked for them (the rest of q's are operands read as
// COUNT columns, and a median's operand has MIN | MAX added); oq: plan_operand_query's.
ScanLayout plan_layout(const tskv_query *q, bool sliding, uint64_t n_cells, uint64_t kern_cells, const tskv_agg_column *user_cols,
                       uint32_t n_user, const OperandQuery &oq) {
  ScanLayout out;
  const StatePlan win = plan_state(q, n_cells, oq.increases);
  const StatePlan pane = sliding ? plan_state(q, kern_cells) : StatePlan{};
  out.sl = win.sl;
  out.kern_sl = sliding ? pane.sl : win.sl;
  out.cols = sliding ? pane.cols : win.cols;
  out.means = win.means;
  out.m2 = win.m2;  // (sliding scans refuse M2)
  out.m2_words = win.m2_words;
  out.pairs = oq.pairs;  // (sliding scans refuse pairs and medians)
  for (size_t p = 0; p < out.pairs.size(); p++) out.pairs[p].off = win.pair_off + (uint64_t)PAIR_WORDS * n_cells * p;
  out.pair_words = win.pair_words;
  out.medians = oq.medians;
  for (size_t m = 0; m < out.medians.size(); m++) {
    MedianCol &mc = out.medians[m];
    mc.count_off = win.cols[mc.qcol].count_off;
    mc.min_off = win.cols[mc.qcol].min_off;
    mc.max_off = win.cols[mc.qcol].max_off;
    mc.off = (uint64_t)MEDIAN_WORDS * n_cells * m;
    mc.hist_off = (uint64_t)MEDIAN_BINS * n_cells * m;
  }
  out.increases = oq.increases;  // (sliding scans refuse increases)
  for (size_t k = 0; k < out.increases.size(); k++) {
    out.increases[k].count_off = win.cols[out.increases[k].qcol].count_off;
    out.increases[k].off = win.inc_off[k];
  }
  if (sliding) {
    for (uint32_t c = 0; c < q->n_columns; c++) {
      const ColState &p = pane.cols[c], &w = win.cols[c];
      const uint8_t m = q->columns[c].agg_mask;
      out.combine.push_back(CombineOp{p.count_off, w.count_off, 0, 0, COMBINE_ADD, 0});
      if (m & (TSKV_AGG_SUM | TSKV_AGG_MEAN)) {
        if (q->columns[c].phys_type == TSKV_PT_F64) out.combine.push_back(CombineOp{p.sum_off, w.sum_off, 0, 0, COMBINE_F64_SUM, 0});
        else out.combine.push_back(CombineOp{p.sum_off, w.sum_off, p.sumhi_off, w.sumhi_off, COMBINE_INT_SUM, (m & TSKV_AGG_MEAN) ? 1u : 0u});
      }
      if (m & TSKV_AGG_MIN) out.combine.push_back(CombineOp{p.min_off, w.min_off, 0, 0, COMBINE_MIN, 0});
      if (m & TSKV_AGG_MAX) out.combine.push_back(CombineOp{p.max_off, w.max_off, 0, 0, COMBINE_MAX, 0});
    }
  }

  // output column table
  uint64_t fk = out.sl.first_keys_off, lk = out.sl.last_keys_off, fv = out.sl.selval_off, lv = out.sl.selval_off + out.sl.first_cells;
  for (uint32_t c = 0; c < n_user; c++) {
    const tskv_agg_column &qc = user_cols[c];
    for (unsigned bit = 0; bit < 8; bit++) {
      unsigned agg = 1u << bit;
      if (!(qc.agg_mask & agg)) continue;
      OutCol oc{};
      oc.count_off = win.cols[c].count_off;
      oc.agg = (uint8_t)agg;
      oc.phys_type = qc.phys_type;
      switch (agg) {
        case TSKV_AGG_SUM: oc.src_off = win.cols[c].sum_off; break;
        case TSKV_AGG_MEAN: oc.src_off = win.msum_off[c] ? win.msum_off[c] : win.cols[c].sum_off; break;
        case TSKV_AGG_MIN: oc.src_off = win.cols[c].min_off; break;
        case TSKV_AGG_MAX: oc.src_off = win.cols[c].max_off; break;
        case TSKV_AGG_FIRST: oc.src_off = fk; oc.val_off = fv; break;
        case TSKV_AGG_LAST: oc.src_off = lk; oc.val_off = lv; break;
        case TSKV_AGG_M2: oc.src_off = win.m2[win.m2_of[c]].sd2_off; oc.val_off = win.m2[win.m2_of[c]].sd_off; break;
        default: break;
      }
      out.outs.push_back(oc);
    }
    if (qc.agg_mask & TSKV_AGG_FIRST) { fk += n_cells; fv += n_cells; }
    if (qc.agg_mask & TSKV_AGG_LAST) { lk += n_cells; lv += n_cells; }
  }

  // per-CTA shared-memory partial table (GROUP BY bucket / tags): count | sum | hi | min | max per column
  std::vector<ColState> &cols = out.cols;
  uint32_t words = 0;
  for (uint32_t c = 0; c < q->n_columns; c++) {
    const uint8_t m = kernel_mask(q->columns[c].agg_mask);
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
  out.use_smem = (!q->group_by_series && (uint64_t)words * 8 <= limit) ? 1u : 0u;
  out.smem_words = out.use_smem ? words : 0;
  // pass 2: count_off = the shifts, sum_off / sumhi_off = sum(d) / sum(d^2); s_sum / s_hi in its own table
  uint64_t words2 = 0;
  for (uint32_t c = 0; c < q->n_columns && !out.m2.empty(); c++) {
    ColState cs{};
    cs.column_id = q->columns[c].column_id;
    cs.phys_type = q->columns[c].phys_type;
    if (win.m2_of[c] >= 0) {
      const M2Col &mc = win.m2[win.m2_of[c]];
      cs.agg_mask = TSKV_AGG_M2;
      cs.count_off = mc.shift_off;
      cs.sum_off = mc.sd_off;
      cs.sumhi_off = mc.sd2_off;
      cs.s_sum = (uint32_t)std::min<uint64_t>(words2, UINT32_MAX);
      cs.s_hi = (uint32_t)std::min<uint64_t>(words2 + kern_cells, UINT32_MAX);
      words2 += 2 * kern_cells;
    }
    out.cols2.push_back(cs);
  }
  out.use_smem2 = (!out.m2.empty() && !q->group_by_series && words2 * 8 <= limit) ? 1u : 0u;
  out.smem_words2 = out.use_smem2 ? (uint32_t)words2 : 0;
  return out;
}

// Parts per page, resident CTAs per SM and grid of every bin's fused kernel (grid 0: the bin is not launched).
void plan_grids(const tskv_ctx *ctx, const tskv_pages *pages, const tskv_query *q, bool has_sel, bool edges, uint32_t smem_words,
                uint32_t has_tomb, int grid[N_BINS], int occ[N_BINS], uint32_t parts[N_BINS], uint32_t part_rows[N_BINS]) {
  for (int b = 0; b < N_BINS; b++) { grid[b] = occ[b] = 0; parts[b] = 1; part_rows[b] = 0; }
  const double sel_frac = plan_selected_fraction(pages->series.data(), pages->series.size(), q->series_ids, q->n_series);
  // Grid sizes. Every kernel is persistent (warps pull tasks from their bin's counter). If the resident
  // capacity allows, each bin gets one warp per estimated task (a single round: the makespan of a bin is
  // quantised in units of one task = one chunk's serial decode); otherwise plan_serial_grids splits the blocks.
  // Pages cut at restart points (skip_kernels.cuh): a chunk of 32 whole pages is one serial task of ~1000 rows; with
  // few selected pages that chain is the scan's makespan, and with many the makespan is still quantised in chunk
  // times. Cut the pages of the simple8b / gorilla bins into parts so that the scan has about 8 chunks per resident
  // warp (more parts = shorter chains, but one more page open + two more run flushes per part).
  // With every bin at 4 CTAs per SM, 8 chunks per resident warp measured best on C4 (H100: 4 parts of 256 rows per
  // 1000-row page instead of 3 uneven parts of 384 / 384 / 232 rows at a target of 4; DESIGN.md §5). The
  // simple8b-timestamp bins take the same parts although their rows cost ~1.6 x the rows of RLE-timestamp pages: twice
  // the parts changed nothing (H100, C4: 1.03-1.05 vs 1.02 ms per scan).
  if (pages->d_skip && !has_sel) {
    double est_chunks = 0;
    for (int b = 0; b < N_BINS; b++) est_chunks += std::ceil(pages->h_bin_pages[b] * sel_frac / 32.0);
    const double resident_warps = (double)ctx->sm_count * SCAN_MIN_BLOCKS * (SCAN_THREADS / 32);
    uint32_t want = plan_parts_wanted(est_chunks, resident_warps, 8.0);
    const char *parts_env = getenv("TSKV_PARTS");  // fixed number of parts (1 = never cut)
    if (parts_env) want = (uint32_t)std::max(1, atoi(parts_env));
    for (int b = 0; b < N_BINS; b++) {
      const int sb = serial_bin_of(b);
      if (sb / N_VK == TK_GEN || sb % N_VK == VK_GEN) continue;
      parts[b] = plan_bin_parts(pages->h_bin_maxrows[b], SKIP_ROWS, want, &part_rows[b]);
    }
  }
  double need_sum = 0, occ_weighted = 0;
  int need[N_BINS] = {0};
  for (int b = 0; b < N_BINS; b++) {
    uint32_t n_bin = pages->h_bin_pages[b];
    if (!n_bin) continue;
    const int sb = serial_bin_of(b);
    const void *fn = (const void *)(!has_sel ? scan_kernel_for<false>(sb, edges, pages->h_bin_narrow[b]) : scan_kernel_for<true>(sb, edges));
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ[b], fn, SCAN_THREADS, serial_smem_bytes(sb, smem_words, has_tomb));
    occ[b] = std::max(1, occ[b]);
    // (an estimate: the work list rounds each (column, narrow flag) bucket of the bin up to 32 items on its own, so the bin
    // may run up to n_cols * WL_SUB - 1 chunks more than items / 32; the kernels are persistent and take them all)
    const double est_items = n_bin * sel_frac * 1.02 + 32;
    const uint32_t per_task = 32;  // pages per warp task: one chunk
    const double tasks = est_items / per_task * parts[b];
    need[b] = (int)(tasks / (SCAN_THREADS / 32)) + 1;
    need[b] = std::min(need[b], (int)(((uint64_t)(n_bin + per_task - 1) / per_task * parts[b] + SCAN_THREADS / 32 - 1) / (SCAN_THREADS / 32)));
    need_sum += need[b];
    occ_weighted += (double)need[b] * occ[b];
  }
  const double capacity = need_sum > 0 ? (occ_weighted / need_sum) * ctx->sm_count : 0;  // resident blocks, mixed kernels
  if (need_sum <= capacity) {
    for (int b = 0; b < N_BINS; b++)
      if (need[b]) grid[b] = std::max(1, need[b]);
    return;
  }
  // a chunk of 32 pages is one long serial task, so a bin's time is quantised in rounds of its chunk time - choose
  // the grids that minimise the makespan (plan_serial_grids)
  double chunks[N_BINS], t_chunk[N_BINS];
  for (int b = 0; b < N_BINS; b++) {
    const uint32_t n_bin = pages->h_bin_pages[b];
    chunks[b] = need[b] ? std::ceil((n_bin * sel_frac * 1.02 + 16) / 32.0) * parts[b] : 0;
    // (+ 12 rows' worth per chunk for opening its pages)
    t_chunk[b] = n_bin ? chunk_cost(b) * ((double)pages->h_bin_rows[b] / n_bin / parts[b] + 12.0) : 1.0;
  }
  plan_serial_grids(N_BINS, chunks, t_chunk, occ, ctx->sm_count, SCAN_THREADS / 32, grid);
  for (int b = 0; b < N_BINS; b++) grid[b] = std::min(grid[b], std::max(need[b], 0));
  // The planned blocks per bin x 4, at most one warp per chunk: the blocks that are not resident at first start as the
  // bins that finish early retire theirs and pick up what is left of the slower bins' chunks.
  // H100, C4 at N = 1 (pages cut in 3 parts), ms per scan: planned grids 1.43-1.50, 2 x 1.10, 4 x 1.02 = one warp per
  // chunk 1.02-1.03. Uncut pages too: planned grids 1.26-1.34, 4 x 1.12; FIRST / LAST scans (C5 shape) and
  // host-resident page sets are the same with either (31.0-31.7 ms).
  for (int b = 0; b < N_BINS; b++) grid[b] = std::min(std::max(need[b], 0), 4 * grid[b]);
}

// The merge pass over the overlapping chunks (merge_kernels.cuh) of one scan: which merge column groups it reads
// (series selected, not pruned by its time bounds), the field pages of the query's columns to decode for them and where
// their values / validity bits go, and the pass's share of the reader counters.
struct MergePages {
  std::vector<uint8_t> active;
  std::vector<uint32_t> page;
  std::vector<uint64_t> row_off, bm_off;
  uint64_t bytes = 0, read_pages = 0;
};
// Refuses (TSKV_ERR_INVALID_ARG, with the page) a page whose type does not match its query column.
tskv_status plan_merge_pages(tskv_ctx *ctx, const tskv_pages *pages, const tskv_query *q, MergePages *m) {
  const OverlapTables &ov = pages->overlap;
  const OverlapPlan &op = ov.plan;
  m->active.assign(op.mcg_cg.size(), 0);
  for (size_t k = 0; k < op.mcg_cg.size(); k++) {
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
            return TSKV_ERR_INVALID_ARG;
          }
          any = true;
          m->page.push_back((uint32_t)p);
          m->row_off.push_back((uint64_t)c * ov.merge_rows + op.mcg_row0[k]);
          m->bm_off.push_back(((uint64_t)c * ov.merge_bm_words + ov.h_mcg_bm0[k]) * 4);
          m->bytes += pages->h_descs[p].size;
        }
    if (!any) continue;  // a column group without any projected column yields no batch (column_group/mod.rs:43-52)
    m->active[k] = 1;
    m->bytes += td.size;
    m->read_pages++;
  }
  m->read_pages += m->page.size();
  return TSKV_OK;
}

// Creates the scan's events, allocates its device buffers (stream-ordered) and uploads the query's tables; sets the
// error. *h2d: the bytes uploaded.
tskv_status alloc_scan(tskv_ctx *ctx, const tskv_pages *pages, const tskv_query *q, const TagGroups &tg, bool sliding,
                       const BucketEdges &E, const ScanLayout &lay, tskv_scan *s, uint64_t *h2d) {
  const uint32_t n_items = pages->n_items;
  cudaStream_t st = ctx->stream.get();
  s->ev0 = new_event();
  s->ev1 = new_event();
  for (int b = 0; b <= N_BINS; b++) s->ev_bin[b] = new_event();
  for (int b = 0; b < N_BINS; b++) {
    s->ev_bin_start[b] = new_event();
    s->ev_bin_done[b] = new_event();
    s->ev_gather[b] = new_event(cudaEventDisableTiming);
  }
  s->n_series_sel = q->series_ids ? q->n_series : 0;
  cudaError_t e = cudaSuccess;
  if (q->series_ids) {
    e = upload(s->d_series, q->series_ids, q->n_series, st);
    *h2d += (uint64_t)q->n_series * 4;
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
    if (e == cudaSuccess) e = upload(s->d_slot_group, tg.ids, n_slots, st);
    if (e == cudaSuccess && !walk.empty()) e = upload(s->d_walk, walk.data(), n_slots, st);
    *h2d += (n_slots + walk.size()) * 4;
  }
  if (E.on) {  // explicit time-bucket edges (params.edges), then the labels of a labelled scan (bucket_cell)
    std::vector<int64_t> table(E.edges, E.edges + (size_t)E.n + 1);
    if (E.labelled) {
      table.resize(table.size() + ((size_t)E.n + 1) / 2);
      std::memcpy(table.data() + E.n + 1, E.labels, (size_t)E.n * 4);
    }
    if (e == cudaSuccess) e = upload(s->d_edges, table.data(), table.size(), st);
    *h2d += ((uint64_t)E.n + 1) * 8 + (E.labelled ? (uint64_t)E.n * 4 : 0);
  }
  if (e == cudaSuccess && q->series_ids) e = stream_alloc(s->d_rank_slot, pages->series.size(), st);
  // work-list regions: each (bin, query column, narrow flag) bucket holds as many items as the page set has field pages
  // of the column's id in that bin with that flag (a later query column with the same id gets no items: find_qcol)
  const uint32_t n_buckets = N_BINS * q->n_columns * WL_SUB;
  s->split_narrow = std::any_of(pages->h_bin_narrow, pages->h_bin_narrow + N_BINS, [](uint8_t m) { return m == NARROW_SOME; });
  std::vector<uint32_t> capacity(n_buckets, 0), region(n_buckets + 1);
  for (uint32_t c = 0; c < q->n_columns; c++) {
    const uint16_t id = q->columns[c].column_id;
    const auto it = pages->col_bucket_pages.find(id);
    if (it == pages->col_bucket_pages.end() ||
        std::any_of(q->columns, q->columns + c, [&](const tskv_agg_column &o) { return o.column_id == id; }))
      continue;
    for (int b = 0; b < N_BINS; b++) {
      const uint32_t k = (b * q->n_columns + c) * WL_SUB, wide = it->second[b * WL_SUB], narrow = it->second[b * WL_SUB + 1];
      capacity[k] = s->split_narrow ? wide : wide + narrow;  // (without the split every item takes the wide bucket)
      capacity[k + 1] = s->split_narrow ? narrow : 0;
    }
  }
  if (!plan_worklist_regions(n_buckets, capacity.data(), region.data())) {
    ctx->set_error("work list too large for 32-bit item indices");
    return TSKV_ERR_INVALID_ARG;
  }
  if (e == cudaSuccess) e = stream_alloc(s->d_bucket, n_buckets, st);
  if (e == cudaSuccess) e = upload(s->d_region, region.data(), region.size(), st);
  {
    // A series with thousands of column groups (one host over a year) is walked by several threads
    const uint64_t n_walk = q->series_ids ? q->n_series : pages->series.size();
    const uint32_t split = plan_walk_split(pages->max_series_cg, n_walk, n_items, WL_THREADS);
    while ((1u << s->walk_split_log2) < split) s->walk_split_log2++;
  }
  if (e == cudaSuccess) e = stream_alloc(s->d_cg_slot, pages->n_cg, st);
  if (e == cudaSuccess) e = stream_alloc(s->d_work_page, region[n_buckets], st);
  if (e == cudaSuccess) e = stream_alloc(s->d_work_slot, region[n_buckets], st);
  if (e == cudaSuccess) e = stream_alloc(s->d_work_qcol, region[n_buckets], st);
  if (e == cudaSuccess) e = upload(s->d_cols, lay.cols.data(), lay.cols.size(), st);
  if (e == cudaSuccess) e = upload(s->d_outs, lay.outs.data(), lay.outs.size(), st);
  s->n_means = (uint32_t)lay.means.size();
  if (e == cudaSuccess) e = upload(s->d_means, lay.means.data(), lay.means.size(), st);
  if (e == cudaSuccess) e = stream_alloc(s->d_state, s->sl.total, st);
  if (e == cudaSuccess && sliding) e = stream_alloc(s->d_pane_state, s->kern_sl.total, st);
  s->n_combine = (uint32_t)lay.combine.size();
  if (e == cudaSuccess && sliding) e = upload(s->d_combine, lay.combine.data(), lay.combine.size(), st);
  s->preds.n = q->n_predicates;
  for (uint32_t k = 0; k < q->n_predicates; k++) s->preds.p[k] = q->predicates[k];
  if (q->n_predicates) ensure_page_stats(ctx, pages);  // value-statistics pruning (filter_column_groups, reader/chunk.rs:12-50)
  if (e == cudaSuccess && q->n_predicates) e = stream_alloc(s->d_row_keep, (size_t)pages->keep_words, st);
  s->n_m2 = (uint32_t)lay.m2.size();
  s->m2_words = lay.m2_words;
  if (s->n_m2) {
    s->ev_m2_fork = new_event(cudaEventDisableTiming);
    for (int b = 0; b < N_BINS; b++) s->ev_m2_join[b] = new_event(cudaEventDisableTiming);
    if (e == cudaSuccess) e = upload(s->d_m2, lay.m2.data(), lay.m2.size(), st);
    if (e == cudaSuccess) e = upload(s->d_cols2, lay.cols2.data(), lay.cols2.size(), st);
    if (e == cudaSuccess) e = stream_alloc(s->d_fill2, (size_t)n_buckets + N_BINS, st);
    *h2d += lay.m2.size() * sizeof(M2Col) + lay.cols2.size() * sizeof(ColState);
    for (uint32_t c = 0; c < q->n_columns; c++) {  // the bins holding pages of an M2 column
      const auto it = pages->col_bucket_pages.find(q->columns[c].column_id);
      if (!(q->columns[c].agg_mask & TSKV_AGG_M2) || it == pages->col_bucket_pages.end()) continue;
      for (int b = 0; b < N_BINS; b++) s->m2_bin[b] |= (it->second[b * WL_SUB] + it->second[b * WL_SUB + 1]) != 0;
    }
  }
  s->n_pairs = (uint32_t)lay.pairs.size();
  s->pair_words = lay.pair_words;
  if (e == cudaSuccess && s->n_pairs) e = upload(s->d_pairs, lay.pairs.data(), lay.pairs.size(), st);
  *h2d += lay.pairs.size() * sizeof(PairCol);
  s->n_medians = (uint32_t)lay.medians.size();
  if (s->n_medians) {  // (the histograms start cleared; every selection step clears the bins it read)
    const uint64_t n_cells = s->layout.n_cells;
    if (e == cudaSuccess) e = upload(s->d_medians, lay.medians.data(), lay.medians.size(), st);
    if (e == cudaSuccess) e = stream_alloc(s->d_med_state, (size_t)MEDIAN_WORDS * n_cells * s->n_medians + 1, st);
    if (e == cudaSuccess) e = stream_alloc(s->d_med_hist, (size_t)MEDIAN_BINS * n_cells * s->n_medians, st);
    if (e == cudaSuccess) e = cudaMemsetAsync(s->d_med_hist.get(), 0, (size_t)MEDIAN_BINS * n_cells * s->n_medians * 4, st);
    s->med.state = s->d_med_state.get();
    s->med.hist = s->d_med_hist.get();
    s->med.unresolved = reinterpret_cast<unsigned long long *>(s->d_med_state.get() + (size_t)MEDIAN_WORDS * n_cells * s->n_medians);
    *h2d += lay.medians.size() * sizeof(MedianCol);
  }
  s->n_increases = (uint32_t)lay.increases.size();
  if (s->n_increases) {
    s->n_inc_merge_rows = pages->overlap.merge_rows;
    // records: each increase's operand items, bucket by bucket (rec0), then the merge rows
    std::vector<uint32_t> rec0((size_t)s->n_increases * N_BINS * WL_SUB);
    uint64_t n_items_max = 0;
    for (uint32_t m = 0; m < s->n_increases; m++) {
      uint64_t acc = 0;
      for (int b = 0; b < N_BINS; b++)
        for (uint32_t sub = 0; sub < WL_SUB; sub++) {
          rec0[((size_t)m * N_BINS + b) * WL_SUB + sub] = (uint32_t)acc;
          acc += capacity[(b * q->n_columns + lay.increases[m].qcol) * WL_SUB + sub];
        }
      n_items_max = std::max(n_items_max, acc);
    }
    const uint64_t n_rec = n_items_max + s->n_inc_merge_rows, n = n_rec * s->n_increases;
    if (n >> 31) {
      ctx->set_error("increase: more than 2^31 page and merge-row records");
      return TSKV_ERR_UNSUPPORTED;
    }
    // sort keys: the slot sort reads (increase, slot) bits, and the slot field of a record never has all of its bits set,
    // so an empty record's ~0 sorts after every other; the time sort reads the bits of the page set's time span
    const uint64_t n_slots = selected_slots(pages, q);
    s->inc.slot_bits = 64 - __builtin_clzll(std::max<uint64_t>(n_slots, 1));
    s->inc_slot_sort_bits = (int)s->inc.slot_bits + (s->n_increases > 1 ? 32 - __builtin_clz(s->n_increases - 1) : 0);
    ensure_time_bounds(ctx, pages);
    s->inc.t_base = INT64_MIN;
    s->inc.t_mask = ~0ull;
    s->inc_time_sort_bits = 64;
    if (pages->ts_min <= pages->ts_max && !(pages->ts_min == INT64_MIN && pages->ts_max == INT64_MAX)) {
      const uint64_t span = (uint64_t)pages->ts_max - (uint64_t)pages->ts_min;
      s->inc.t_base = pages->ts_min;
      s->inc_time_sort_bits = span ? 64 - __builtin_clzll(span) : 1;
      s->inc.t_mask = s->inc_time_sort_bits == 64 ? ~0ull : (1ull << s->inc_time_sort_bits) - 1;
    }
    size_t t1 = 0, t2 = 0;
    if (e == cudaSuccess) e = cub::DeviceRadixSort::SortPairs(nullptr, t1, (const uint64_t *)nullptr, (uint64_t *)nullptr, (const uint32_t *)nullptr,
                                                               (uint32_t *)nullptr, (int)n, 0, s->inc_time_sort_bits, st);
    if (e == cudaSuccess) e = cub::DeviceRadixSort::SortPairs(nullptr, t2, (const uint64_t *)nullptr, (uint64_t *)nullptr, (const uint32_t *)nullptr,
                                                               (uint32_t *)nullptr, (int)n, 0, s->inc_slot_sort_bits, st);
    s->inc_tmp_bytes = std::max<size_t>(std::max(t1, t2), 1);
    if (e == cudaSuccess) e = upload(s->d_increases, lay.increases.data(), lay.increases.size(), st);
    if (e == cudaSuccess) e = stream_alloc(s->d_inc_rec, (size_t)std::max<uint64_t>(n, 1), st);
    if (e == cudaSuccess) e = stream_alloc(s->d_inc_keys, (size_t)std::max<uint64_t>(5 * n, 1), st);
    if (e == cudaSuccess) e = stream_alloc(s->d_inc_idx, (size_t)std::max<uint64_t>(3 * n, 1), st);
    if (e == cudaSuccess) e = stream_alloc(s->d_inc_tmp, s->inc_tmp_bytes, st);
    if (e == cudaSuccess) e = upload(s->d_inc_rec0, rec0.data(), rec0.size(), st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);  // (rec0 goes out of scope)
    s->inc.rec = s->d_inc_rec.get();
    s->inc.rec0 = s->d_inc_rec0.get();
    s->inc.slot_key = s->d_inc_keys.get();
    s->inc.time_key = s->d_inc_keys.get() + n;
    s->inc.n_rec = (uint32_t)n_rec;
    *h2d += lay.increases.size() * sizeof(IncreaseCol) + rec0.size() * 4;
  }
  if (e == cudaSuccess) e = stream_alloc(s->d_aux, AUX_WORDS, st);
  if (e == cudaSuccess) e = stream_alloc(s->d_values, s->layout.n_out * s->layout.n_cells, st);
  if (e == cudaSuccess) e = stream_alloc(s->d_validity, s->layout.validity_bytes + 8, st);
  *h2d += lay.cols.size() * sizeof(ColState) + lay.outs.size() * sizeof(OutCol) + lay.means.size() * sizeof(MeanExport) +
          sizeof(ScanParams) + lay.combine.size() * sizeof(CombineOp);
  if (e != cudaSuccess) {
    ctx->set_error(std::string("scan_prepare: ") + cudaGetErrorString(e));
    return e == cudaErrorMemoryAllocation ? TSKV_ERR_OOM : TSKV_ERR_CUDA;
  }
  unsigned long long *aux = s->d_aux.get();
  s->d_status = reinterpret_cast<int32_t *>(aux + AUX_STATUS);
  s->d_err_page = aux + AUX_ERR_PAGE;
  s->d_stats = aux + AUX_STATS;
  s->d_counters = aux + AUX_COUNTERS;
  s->d_crc_status = reinterpret_cast<int32_t *>(aux + AUX_CRC_STATUS);
  s->d_crc_err_page = aux + AUX_CRC_ERR_PAGE;
  return TSKV_OK;
}

// The merge pass of a scan over a page set with overlapping chunks: its page list on the device and s->merge; sets the
// error. *h2d: the bytes uploaded.
tskv_status prepare_merge(tskv_ctx *ctx, const tskv_pages *pages, const tskv_query *q, tskv_scan *s, uint64_t *h2d) {
  MergePages mp;
  const tskv_status st = plan_merge_pages(ctx, pages, q, &mp);
  if (st != TSKV_OK) return st;
  const size_t n_mcg = mp.active.size(), n_mpages = mp.page.size();
  s->n_merge_pages = (uint32_t)n_mpages;
  s->merge_page_bytes = mp.bytes;
  s->merge_read_pages = mp.read_pages;
  const OverlapTables &ov = pages->overlap;
  cudaStream_t stream = ctx->stream.get();
  cudaError_t e = upload(s->d_mcg_active, mp.active.data(), n_mcg, stream);
  if (e == cudaSuccess) e = stream_alloc(s->d_mvals, (size_t)q->n_columns * ov.merge_rows, stream);
  if (e == cudaSuccess) e = stream_alloc(s->d_mvalid, (size_t)q->n_columns * ov.merge_bm_words, stream);
  if (e == cudaSuccess) e = upload(s->d_mpage, mp.page.data(), n_mpages, stream);
  if (e == cudaSuccess) e = upload(s->d_mrow_off, mp.row_off.data(), n_mpages, stream);
  if (e == cudaSuccess) e = upload(s->d_mbm_off, mp.bm_off.data(), n_mpages, stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(stream);  // the host vectors go out of scope
  if (e != cudaSuccess) {
    ctx->set_error(std::string("scan_prepare (merge pass): ") + cudaGetErrorString(e));
    return e == cudaErrorMemoryAllocation ? TSKV_ERR_OOM : TSKV_ERR_CUDA;
  }
  *h2d += n_mcg + n_mpages * 20;
  MergeParams &M = s->merge;
  M.ts = ov.d_merge_ts.get();
  M.mcg_row0 = ov.d_mcg_row0.get();
  M.mcg_cg = ov.d_mcg_cg.get();
  M.mcg_stream = ov.d_mcg_stream.get();
  M.stream_group = ov.d_stream_group.get();
  M.stream_first_mcg = ov.d_stream_first_mcg.get();
  M.group_first_stream = ov.d_group_first_stream.get();
  M.mcg_active = s->d_mcg_active.get();
  M.vals = s->d_mvals.get();
  M.valid = s->d_mvalid.get();
  M.mcg_bm0 = ov.d_mcg_bm0.get();
  M.cg_time_page = pages->d_cg_time_page.get();
  M.cg_slot = s->d_cg_slot.get();
  M.n_rows = ov.merge_rows;
  M.bm_words = ov.merge_bm_words;
  M.n_mcg = (uint32_t)n_mcg;
  M.sel = s->has_sel ? 1u : 0u;
  return TSKV_OK;
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
  cudaStreamSynchronize(ctx->stream.get());
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
  cudaStream_t st = nullptr;
  const bool ok = cudaSetDevice(device_id) == cudaSuccess && cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking) == cudaSuccess;
  ctx->stream.reset(ok ? st : nullptr);
  if (!ok || !(ctx->ev0 = new_event()) || !(ctx->ev1 = new_event())) {
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
      cudaStream_t bs = nullptr;
      if (cudaStreamCreateWithPriority(&bs, cudaStreamNonBlocking, prio) != cudaSuccess)
        cudaStreamCreateWithFlags(&bs, cudaStreamNonBlocking);
      ctx->bin_stream[b].reset(bs);
    }
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
      for (const bool edges : {false, true}) {
        for (int nm = NARROW_NONE; nm <= NARROW_ALL; nm++) raise((const void *)scan_kernel_for<false>(b, edges, nm));
        raise((const void *)scan_kernel_for<true>(b, edges));
        raise((const void *)m2_kernel_for(b, edges));
      }
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
  if (ctx->stream) cudaStreamSynchronize(ctx->stream.get());
  delete ctx;
}

const char *tskvgpu_last_error(const tskv_ctx *ctx) { return ctx ? ctx->err.c_str() : "null context"; }
int64_t tskvgpu_last_error_page(const tskv_ctx *ctx) { return ctx ? ctx->err_page : -1; }
tskv_status tskvgpu_get_counters(const tskv_ctx *ctx, tskv_counters *out) {
  if (!ctx || !out) return TSKV_ERR_INVALID_ARG;
  *out = ctx->counters;
  return TSKV_OK;
}
uint64_t tskvgpu_ctx_stream(const tskv_ctx *ctx) { return ctx ? (uint64_t)(uintptr_t)ctx->stream.get() : 0; }

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
  std::unique_ptr<tskv_pages> pg(new tskv_pages());
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
    return st;
  }

  // ---- column groups ----------------------------------------------------------------------------
  std::vector<uint32_t> time_page_of(n_descs, 0), cg_time_page;
  {
    uint64_t i = 0;
    while (i < n_descs) {
      if (pg->h_descs[i].phys_type != TSKV_PT_TIME) {
        ctx->set_error("descriptor table: column group does not start with a time page", (int64_t)i);
        return TSKV_ERR_INVALID_ARG;
      }
      cg_time_page.push_back((uint32_t)i);
      time_page_of[i] = (uint32_t)i;
      uint64_t j = i + 1;
      while (j < n_descs && pg->h_descs[j].phys_type != TSKV_PT_TIME) {
        if (pg->h_descs[j].series_id != pg->h_descs[i].series_id || pg->h_descs[j].num_values != pg->h_descs[i].num_values) {
          ctx->set_error("descriptor table: field page disagrees with its time page", (int64_t)j);
          return TSKV_ERR_INVALID_ARG;
        }
        time_page_of[j] = (uint32_t)i;
        j++;
      }
      i = j;
    }
  }
  pg->n_cg = (uint32_t)cg_time_page.size();
  pg->n_items = (uint32_t)(n_descs - cg_time_page.size());
  pg->h_cg_time_page = cg_time_page;
  pg->h_time_has_nulls = time_has_nulls;
  std::vector<uint32_t> keep_off(n_descs, 0);
  for (uint32_t tp : cg_time_page) {
    keep_off[tp] = (uint32_t)pg->keep_words;
    pg->keep_words += ((uint64_t)pg->h_descs[tp].num_values + 31) / 32;
  }
  if (pg->keep_words >= (1ull << 32)) {
    ctx->set_error("too many rows for one arena (2^37)");
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
  // decode-kind bin of every field page, and the bins' page counts, bytes, rows and longest pages
  std::vector<uint8_t> page_bin(n_descs, 0);
  for (uint64_t p = 0; p < n_descs; p++) {
    const tskv_page_desc &vd = pg->h_descs[p];
    if (vd.phys_type == TSKV_PT_TIME) continue;
    const int tclass = time_has_nulls[time_page_of[p]] ? TK_GEN : time_class(pg->h_descs[time_page_of[p]].reserved);
    int bin = tclass * N_VK + value_class(vd.reserved);
    if (vd.num_values <= SHORT_PAGE_ROWS && vd.reserved == DK_S8B_ZZ && tclass != TK_GEN)
      bin = tclass == TK_RLE ? BIN_SHORT_RLE_S8B : BIN_SHORT_S8B_S8B;
    if (vd.num_values <= SHORT_PAGE_ROWS && vd.reserved == DK_GORILLA && tclass != TK_GEN)
      bin = tclass == TK_RLE ? BIN_SHORT_RLE_GOR : BIN_SHORT_S8B_GOR;
    page_bin[p] = (uint8_t)bin;
    pg->h_bin_pages[bin]++;
    std::vector<uint32_t> &cb = pg->col_bucket_pages[vd.column_id];
    if (cb.empty()) cb.assign(N_BINS * WL_SUB, 0);
    cb[bin * WL_SUB]++;
    pg->h_bin_bytes[bin] += vd.size;
    pg->h_bin_rows[bin] += vd.num_values;
    pg->h_bin_maxrows[bin] = std::max(pg->h_bin_maxrows[bin], vd.num_values);
  }

  // ---- device copies ----------------------------------------------------------------------------
  cudaStream_t st = ctx->stream.get();
  cudaEventRecord(ctx->ev0.get(), st);
  cudaError_t e = dev_alloc(pg->d_arena, arena_len + ARENA_SLACK);
  if (e == cudaSuccess) e = cudaMemsetAsync(pg->d_arena.get() + arena_len, 0, ARENA_SLACK, ctx->stream.get());
  if (e == cudaSuccess && arena_len && (flags & TSKV_UPLOAD_HOST_RESIDENT)) {
    // pages stay in (page-locked) host memory like the reference's page cache; each scan pulls the
    // selected pages over PCIe itself (k_gather_pages)
    e = cudaHostRegister(const_cast<uint8_t *>(arena), arena_len, cudaHostRegisterMapped | cudaHostRegisterPortable);
    if (e == cudaSuccess) pg->h_registered.reset(const_cast<uint8_t *>(arena));
    else if (e == cudaErrorHostMemoryAlreadyRegistered) { cudaGetLastError(); e = cudaSuccess; }
    void *dp = nullptr;
    if (e == cudaSuccess) e = cudaHostGetDevicePointer(&dp, const_cast<uint8_t *>(arena), 0);
    pg->h_mapped = static_cast<const uint8_t *>(dp);
  } else if (e == cudaSuccess && arena_len) {
    e = cudaMemcpyAsync(pg->d_arena.get(), arena, arena_len, cudaMemcpyHostToDevice, ctx->stream.get());
  }
  if (e == cudaSuccess) e = upload(pg->d_descs, pg->h_descs.data(), n_descs, st);
  if (e == cudaSuccess) e = upload(pg->d_time_page_of, time_page_of.data(), n_descs, st);
  if (e == cudaSuccess) e = upload(pg->d_cg_time_page, cg_time_page.data(), pg->n_cg, st);
  if (e == cudaSuccess) e = upload(pg->d_cg_series_rank, cg_rank.data(), pg->n_cg, st);
  if (e == cudaSuccess) e = upload(pg->d_series_sorted, pg->series.data(), pg->series.size(), st);
  if (e == cudaSuccess && plan_series_map(pg->series.empty() ? 0 : pg->series.front(), pg->series.empty() ? 0 : pg->series.back(),
                                          pg->series.size())) {
    pg->series_min = pg->series.front();
    pg->series_span = pg->series.back() - pg->series.front() + 1;
    std::vector<uint32_t> rank_of(pg->series_span, 0xffffffffu);
    for (size_t r = 0; r < pg->series.size(); r++) rank_of[pg->series[r] - pg->series_min] = (uint32_t)r;
    e = upload(pg->d_rank_of, rank_of.data(), rank_of.size(), st);
  }
  {  // series rank -> its column groups (the selection-driven work list walks a selected series' groups)
    std::vector<uint32_t> start(pg->series.size() + 1, 0), list(pg->n_cg);
    for (uint32_t cg = 0; cg < pg->n_cg; cg++) start[cg_rank[cg] + 1]++;
    for (size_t r = 0; r < pg->series.size(); r++) {
      pg->max_series_cg = std::max(pg->max_series_cg, start[r + 1]);
      start[r + 1] += start[r];
    }
    std::vector<uint32_t> cur(start.begin(), start.end() - 1);
    for (uint32_t cg = 0; cg < pg->n_cg; cg++) list[cur[cg_rank[cg]]++] = cg;
    if (e == cudaSuccess) e = upload(pg->d_rank_cg_start, start.data(), start.size(), st);
    if (e == cudaSuccess) e = upload(pg->d_rank_cg, list.data(), list.size(), st);
    if (e == cudaSuccess) e = upload(pg->d_page_bin, page_bin.data(), n_descs, st);
  }
  if (e == cudaSuccess) e = upload(pg->d_keep_off, keep_off.data(), n_descs, st);
  if (e == cudaSuccess && (((flags & TSKV_UPLOAD_VERIFY_CRC) && (flags & TSKV_UPLOAD_HOST_RESIDENT)) || (flags & TSKV_UPLOAD_VERIFY_ON_READ))) {
    pg->verify_on_read = true;  // like the reference: every read of a page re-checks its CRC (device side)
    e = upload(pg->d_crc_tables, crc32_tables(), 2048, st);
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
      e = dev_alloc(pg->d_narrow, n_descs);
      if (e == cudaSuccess) e = cudaMemsetAsync(pg->d_narrow.get(), 0, n_descs, st);
    }
    if (n_skip) {
      pg->n_skip = n_skip;
      if (e == cudaSuccess) e = upload(pg->d_skip_off, skip_off.data(), n_descs, st);
      if (e == cudaSuccess) e = dev_alloc(pg->d_skip, n_skip);
    }
    const size_t n_list = list[0].size() + list[1].size() + list[2].size();
    if (n_list) {
      async_ptr<uint32_t> d_list;  // freed on the stream after the kernels that read it
      if (e == cudaSuccess) e = stream_alloc(d_list, n_list, st);
      size_t lo = 0;
      for (int k = 0; k < 3 && e == cudaSuccess; k++) {
        const uint32_t n = (uint32_t)list[k].size();
        if (!n) continue;
        e = cudaMemcpyAsync(d_list.get() + lo, list[k].data(), (size_t)n * 4, cudaMemcpyHostToDevice, st);
        if (e != cudaSuccess) break;
        const uint32_t blocks = (n + SKIP_THREADS - 1) / SKIP_THREADS;
        if (k == SKIP_KIND_TIME_S8B)
          k_build_skip<SKIP_KIND_TIME_S8B><<<blocks, SKIP_THREADS, SKIP_SMEM_BYTES, ctx->stream.get()>>>(pg->d_arena.get(), pg->d_descs.get(), d_list.get() + lo, n, pg->d_skip_off.get(), pg->d_skip.get(), nullptr);
        else if (k == SKIP_KIND_VALUE_S8B)
          k_build_skip<SKIP_KIND_VALUE_S8B><<<blocks, SKIP_THREADS, SKIP_SMEM_BYTES, ctx->stream.get()>>>(pg->d_arena.get(), pg->d_descs.get(), d_list.get() + lo, n, pg->d_skip_off.get(), pg->d_skip.get(), pg->d_narrow.get());
        else
          k_build_skip<SKIP_KIND_VALUE_GORILLA><<<blocks, SKIP_THREADS, SKIP_SMEM_BYTES, ctx->stream.get()>>>(pg->d_arena.get(), pg->d_descs.get(), d_list.get() + lo, n, pg->d_skip_off.get(), pg->d_skip.get(), nullptr);
        lo += n;
      }
      if (e == cudaSuccess) e = cudaGetLastError();
      // the page lists are read by kernels still in flight: host vectors stay alive until the sync below
      if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    }
    if (e == cudaSuccess && pg->d_narrow) {
      std::vector<uint8_t> narrow(n_descs);
      e = cudaMemcpyAsync(narrow.data(), pg->d_narrow.get(), n_descs, cudaMemcpyDeviceToHost, ctx->stream.get());
      if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream.get());
      uint64_t n_narrow[N_BINS] = {0};
      for (uint64_t p = 0; p < n_descs; p++)
        if (pg->h_descs[p].phys_type != TSKV_PT_TIME && narrow[p]) {
          n_narrow[page_bin[p]]++;
          std::vector<uint32_t> &cb = pg->col_bucket_pages[pg->h_descs[p].column_id];
          cb[page_bin[p] * WL_SUB]--;
          cb[page_bin[p] * WL_SUB + 1]++;
        }
      for (int b = 0; b < N_BINS; b++)
        pg->h_bin_narrow[b] = n_narrow[b] == 0 ? NARROW_NONE : n_narrow[b] == pg->h_bin_pages[b] ? NARROW_ALL : NARROW_SOME;
    }
  }
  cudaEventRecord(ctx->ev1.get(), ctx->stream.get());
  if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream.get());
  if (e != cudaSuccess) {
    ctx->set_error(std::string("upload: ") + cudaGetErrorString(e));
    tskvgpu_pages_destroy(nullptr, pg.release());
    return e == cudaErrorMemoryAllocation ? TSKV_ERR_OOM : TSKV_ERR_CUDA;
  }
  float ms = 0;
  cudaEventElapsedTime(&ms, ctx->ev0.get(), ctx->ev1.get());
  ctx->counters.elapsed_h2d_ms = ms;
  *out_pages = pg.release();
  return TSKV_OK;
}

void tskvgpu_pages_destroy(tskv_ctx *ctx, tskv_pages *pg) {
  (void)ctx;
  if (!pg) return;
  if (pg->ctx) cudaSetDevice(pg->ctx->device);
  if (pg->ctx && pg->ctx->stream) cudaStreamSynchronize(pg->ctx->stream.get());
  delete pg;
}

uint64_t tskvgpu_pages_series_count(const tskv_pages *pages) { return pages ? pages->series.size() : 0; }

tskv_status tskvgpu_pages_set_time_bounds(tskv_ctx *ctx, tskv_pages *pg, const tskv_time_range *bounds, uint64_t n) {
  if (!ctx || !pg || !bounds || n != pg->n_cg) return TSKV_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(ctx->mu);
  ctx->set_error("");
  CU_TRY(ctx, cudaSetDevice(ctx->device));
  CU_TRY(ctx, fill_table(pg->d_cg_bounds, bounds, n, ctx->stream.get()));
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
  CU_TRY(ctx, fill_table(pg->d_page_stats, keys.data(), keys.size(), ctx->stream.get()));
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
    CU_TRY(ctx, cudaStreamSynchronize(ctx->stream.get()));
    pg->overlap = OverlapTables{};
    pg->chunk_epoch++;
    if (n_cg == 0) return TSKV_OK;
    ensure_time_bounds(ctx, pg);  // ColumnGroup::time_range() of every group (the caller's, or one pass over the time pages)
    if (!pg->d_cg_bounds) {
      ctx->set_error("set_chunk_files: the column groups' time bounds are not available");
      return TSKV_ERR_CUDA;
    }
    pg->h_cg_bounds.resize(pg->n_cg);
    CU_TRY(ctx, cudaMemcpy(pg->h_cg_bounds.data(), pg->d_cg_bounds.get(), (size_t)pg->n_cg * sizeof(tskv_time_range), cudaMemcpyDeviceToHost));
    std::vector<uint32_t> cg_series(pg->n_cg), cg_rows(pg->n_cg);
    for (uint32_t cg = 0; cg < pg->n_cg; cg++) {
      cg_series[cg] = pg->h_descs[pg->h_cg_time_page[cg]].series_id;
      cg_rows[cg] = pg->h_descs[pg->h_cg_time_page[cg]].num_values;
    }
    // built here and published only when complete: a failed call leaves the page set without an overlap plan
    OverlapTables t;
    plan_overlap_groups(pg->n_cg, cg_series.data(), cg_rows.data(), pg->h_cg_bounds.data(), cg_file_id, &t.plan);
    const OverlapPlan &op = t.plan;
    const size_t n_mcg = op.mcg_cg.size();
    if (n_mcg == 0) {  // no two chunks of a series overlap: nothing to merge
      pg->overlap = std::move(t);
      return TSKV_OK;
    }
    for (uint32_t cg : op.mcg_cg)
      if (pg->h_time_has_nulls[pg->h_cg_time_page[cg]] || dk_is_error(pg->h_descs[pg->h_cg_time_page[cg]].reserved)) {
        ctx->set_error("set_chunk_files: a time page of an overlapping chunk holds NULLs or does not decode", pg->h_cg_time_page[cg]);
        return TSKV_ERR_UNSUPPORTED;
      }
    t.merge_rows = op.mcg_row0.back();
    t.h_mcg_bm0.assign(n_mcg, 0);
    uint64_t w = 0;
    for (size_t k = 0; k < n_mcg; k++) {
      t.h_mcg_bm0[k] = w;
      w += ((op.mcg_row0[k + 1] - op.mcg_row0[k] + 63) / 64) * 2;  // 8-byte padded bitmaps, in 32-bit words
    }
    t.merge_bm_words = w;
    cudaStream_t st = ctx->stream.get();
    cudaError_t e = upload(t.d_cg_merge, op.cg_merge.data(), op.cg_merge.size(), st);
    if (e == cudaSuccess) e = upload(t.d_mcg_row0, op.mcg_row0.data(), op.mcg_row0.size(), st);
    if (e == cudaSuccess) e = upload(t.d_mcg_bm0, t.h_mcg_bm0.data(), t.h_mcg_bm0.size(), st);
    if (e == cudaSuccess) e = upload(t.d_mcg_cg, op.mcg_cg.data(), op.mcg_cg.size(), st);
    if (e == cudaSuccess) e = upload(t.d_mcg_stream, op.mcg_stream.data(), op.mcg_stream.size(), st);
    if (e == cudaSuccess) e = upload(t.d_stream_group, op.stream_group.data(), op.stream_group.size(), st);
    if (e == cudaSuccess) e = upload(t.d_stream_first_mcg, op.stream_first_mcg.data(), op.stream_first_mcg.size(), st);
    if (e == cudaSuccess) e = upload(t.d_group_first_stream, op.group_first_stream.data(), op.group_first_stream.size(), st);
    if (e == cudaSuccess) e = dev_alloc(t.d_merge_ts, (size_t)t.merge_rows);
    // the merge rows' timestamps: the time pages of the merge column groups, decoded in merge-row order
    std::vector<uint32_t> tpages(n_mcg);
    std::vector<uint64_t> row_off(n_mcg), bm_off(n_mcg);
    for (size_t k = 0; k < n_mcg; k++) {
      tpages[k] = pg->h_cg_time_page[op.mcg_cg[k]];
      row_off[k] = op.mcg_row0[k];
      bm_off[k] = t.h_mcg_bm0[k] * 4;
    }
    dev_ptr<uint32_t> d_list;
    dev_ptr<uint64_t> d_ro, d_bo;
    dev_ptr<uint8_t> d_bm;
    dev_ptr<int32_t> d_st;
    if (e == cudaSuccess) e = upload(d_list, tpages.data(), n_mcg, st);
    if (e == cudaSuccess) e = upload(d_ro, row_off.data(), n_mcg, st);
    if (e == cudaSuccess) e = upload(d_bo, bm_off.data(), n_mcg, st);
    if (e == cudaSuccess) e = dev_alloc(d_bm, (size_t)t.merge_bm_words * 4);
    if (e == cudaSuccess) e = dev_alloc(d_st, 8);  // status | err page (2 x 8 bytes) | points
    tskv_status ret = TSKV_OK;
    if (e == cudaSuccess) e = cudaMemsetAsync(d_st.get(), 0, 32, st);
    if (e == cudaSuccess) {
      unsigned long long *aux = reinterpret_cast<unsigned long long *>(d_st.get());
      const uint32_t blocks = (uint32_t)((n_mcg * 32 + DECODE_THREADS - 1) / DECODE_THREADS);
      k_decode_warp<<<blocks, DECODE_THREADS, 0, st>>>(pg->h_mapped ? pg->h_mapped : pg->d_arena.get(), pg->d_descs.get(), 0, d_list.get(),
                                                       (uint32_t)n_mcg, d_ro.get(), d_bo.get(), reinterpret_cast<uint64_t *>(t.d_merge_ts.get()),
                                                       d_bm.get(), d_st.get(), aux + 1, aux + 2);
      e = cudaGetLastError();
      if (e == cudaSuccess) ret = fetch_status(ctx, d_st.get(), aux + 1);
    }
    if (e != cudaSuccess || ret != TSKV_OK) {
      if (e != cudaSuccess) ctx->set_error(std::string("set_chunk_files: ") + cudaGetErrorString(e));
      return e == cudaErrorMemoryAllocation ? TSKV_ERR_OOM : (e != cudaSuccess ? TSKV_ERR_CUDA : ret);
    }
    pg->overlap = std::move(t);
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
  TombTables t;
  t.n_keys = (uint32_t)keys.size();
  t.n_global = n_global;
  t.n_ranges = (uint32_t)ranges.size();
  cudaStream_t st = ctx->stream.get();
  if (!ranges.empty()) {
    CU_TRY(ctx, upload(t.ranges, ranges.data(), ranges.size(), st));
    CU_TRY(ctx, upload(t.keys, keys.data(), keys.size(), st));
    CU_TRY(ctx, upload(t.off, off.data(), off.size(), st));
  }
  CU_TRY(ctx, cudaStreamSynchronize(st));  // the tables are filled and no scan of this page set is in flight
  pg->tomb = std::move(t);
  pg->tomb_epoch++;
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
  cudaStream_t st = ctx->stream.get();
  dev_ptr<uint64_t> d_row_off, d_bm_off, d_vals;
  dev_ptr<uint8_t> d_valid;
  dev_ptr<int32_t> d_status;
  dev_ptr<unsigned long long> d_aux;  // [0] err_page, [1] points
  tskv_status ret = TSKV_OK;
  cudaError_t e = upload(d_row_off, row_off.data(), n_pages, st);
  if (e == cudaSuccess) e = upload(d_bm_off, bm_off.data(), n_pages, st);
  if (e == cudaSuccess) e = dev_alloc(d_vals, rows);
  if (e == cudaSuccess) e = dev_alloc(d_valid, bm);
  if (e == cudaSuccess) e = dev_alloc(d_status, 1);
  if (e == cudaSuccess) e = dev_alloc(d_aux, 2);
  if (e == cudaSuccess) e = cudaMemsetAsync(d_status.get(), 0, 4, st);
  if (e == cudaSuccess) e = cudaMemsetAsync(d_aux.get(), 0, 16, st);
  if (e == cudaSuccess) e = cudaMemsetAsync(d_vals.get(), 0, std::max<uint64_t>(rows, 1) * 8, st);
  if (e == cudaSuccess) {
    cudaEventRecord(ctx->ev0.get(), ctx->stream.get());
    uint32_t blocks = (uint32_t)((n_pages * 32 + DECODE_THREADS - 1) / DECODE_THREADS);  // one warp per page
    // host-resident page sets: d_arena is only the scans' gather target, the pages are read through the mapped host range
    k_decode_warp<<<blocks, DECODE_THREADS, 0, ctx->stream.get()>>>(pages->h_mapped ? pages->h_mapped : pages->d_arena.get(), pages->d_descs.get(), first_page, nullptr, (uint32_t)n_pages,
                                                        d_row_off.get(), d_bm_off.get(), d_vals.get(), d_valid.get(), d_status.get(), d_aux.get(), d_aux.get() + 1);
    cudaEventRecord(ctx->ev1.get(), ctx->stream.get());
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaMemcpyAsync(out_values, d_vals.get(), rows * 8, cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaMemcpyAsync(out_validity, d_valid.get(), bm, cudaMemcpyDeviceToHost, st);
  unsigned long long points = 0;
  if (e == cudaSuccess) e = cudaMemcpyAsync(&points, d_aux.get() + 1, 8, cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) {
    ret = fetch_status(ctx, d_status.get(), d_aux.get());
  } else {
    ctx->set_error(std::string("decode: ") + cudaGetErrorString(e));
    ret = e == cudaErrorMemoryAllocation ? TSKV_ERR_OOM : TSKV_ERR_CUDA;
  }
  if (ret == TSKV_OK) {
    float ms = 0;
    cudaEventElapsedTime(&ms, ctx->ev0.get(), ctx->ev1.get());
    ctx->counters.elapsed_scan_ms = ms;
    ctx->counters.points_decoded = points;
    ctx->counters.kernel_launches = 1;
    ctx->counters.page_read_count = n_pages;
  }
  return ret;
}

// ------------------------------------------------------------------------------------------------
tskv_status tskvgpu_query_output_layout(const tskv_pages *pages, const tskv_query *q,
                                        tskv_output_layout *out) {
  return compute_layout(pages, q, TagGroups{}, BucketEdges{}, out);
}

tskv_status tskvgpu_query_output_layout_grouped(const tskv_pages *pages, const tskv_query *q, const uint32_t *group_ids,
                                                uint32_t n_groups, tskv_output_layout *out) {
  return compute_layout(pages, q, TagGroups{true, group_ids, n_groups}, BucketEdges{}, out);
}

// The edges of the *_edges calls: q->n_buckets edge buckets, which are the output buckets.
static BucketEdges plain_edges(const tskv_query *q, const int64_t *edges) {
  return BucketEdges{true, edges, q ? q->n_buckets : 0u, false, nullptr};
}

tskv_status tskvgpu_query_output_layout_edges(const tskv_pages *pages, const tskv_query *q, const int64_t *edges,
                                              const uint32_t *group_ids, uint32_t n_groups, tskv_output_layout *out) {
  return compute_layout(pages, q, TagGroups{group_ids != nullptr, group_ids, n_groups}, plain_edges(q, edges), out);
}

tskv_status tskvgpu_query_output_layout_labels(const tskv_pages *pages, const tskv_query *q, const int64_t *edges,
                                               uint32_t n_edge, const uint32_t *labels, const uint32_t *group_ids,
                                               uint32_t n_groups, tskv_output_layout *out) {
  return compute_layout(pages, q, TagGroups{group_ids != nullptr, group_ids, n_groups},
                        BucketEdges{true, edges, n_edge, true, labels}, out);
}

// tskvgpu_scan_prepare; slide > 0: tskvgpu_scan_prepare_sliding with slide < width; tg.on: GROUP BY tags; E.on:
// tskvgpu_scan_prepare_edges / _labels (slide 0).
static tskv_status prepare_scan(tskv_ctx *ctx, const tskv_pages *pages, const tskv_query *q, int64_t slide,
                                const TagGroups &tg, tskv_scan **out_scan, const BucketEdges &E = BucketEdges{}) {
  if (!ctx || !pages || !q || !out_scan) return TSKV_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(ctx->mu);
  ctx->set_error("");
  *out_scan = nullptr;
  uint32_t win_k = 1;
  tskv_status st = validate_query(ctx, pages, q, slide, tg, E, &win_k);
  if (st != TSKV_OK) return st;
  const tskv_output_layout L = output_layout(pages, q, tg);
  if (query_n_medians(q) && (uint64_t)query_n_medians(q) * L.n_cells > TSKV_MAX_MEDIAN_CELLS) {
    ctx->set_error("median: more than 2^22 cells times medians (1 KiB of histogram per cell and median)");
    return TSKV_ERR_UNSUPPORTED;
  }
  // column pairs, medians and increases: from here on the scan runs the query with the operands as columns
  // (plan_operand_query)
  const tskv_agg_column *user_cols = q->columns;
  const uint32_t n_user = q->n_columns;
  OperandQuery pq = plan_operand_query(q);
  pq.q.columns = pq.cols.data();
  q = &pq.q;
  cudaSetDevice(ctx->device);
  bool has_sel = false;  // any FIRST / LAST
  for (uint32_t c = 0; c < q->n_columns; c++) has_sel |= (q->columns[c].agg_mask & (TSKV_AGG_FIRST | TSKV_AGG_LAST)) != 0;
  uint32_t slot_bits = 0;
  int64_t rel_base = 0;
  st = plan_keys(ctx, pages, q, E, has_sel, &slot_bits, &rel_base);
  if (st != TSKV_OK) return st;
  tskv_scan *s = new tskv_scan();
  s->ctx = ctx;
  s->pages = pages;
  s->layout = L;
  s->n_cols = q->n_columns;
  s->n_out = (uint32_t)L.n_out;
  s->has_sel = has_sel;
  // the fused kernels' bucket grid: the query's, or for a sliding scan the panes of width `slide`, from the start of the
  // last pane of window 0 to the start of the last window
  s->win_k = win_k;
  s->n_windows = q->n_buckets;
  s->n_panes = q->n_buckets - win_k + 1;
  const ScanLayout lay = plan_layout(q, slide != 0, L.n_cells, L.n_groups * s->n_panes, user_cols, n_user, pq);
  s->n_out = (uint32_t)lay.outs.size();  // (the pairs' outputs follow, k_finalize_pairs, then the medians')
  s->sl = lay.sl;
  s->kern_sl = lay.kern_sl;
  uint64_t h2d = 0;
  if ((st = alloc_scan(ctx, pages, q, tg, slide != 0, E, lay, s, &h2d)) != TSKV_OK) {
    delete s;
    return st;
  }
  ScanParams &P = s->params;
  P.arena = pages->d_arena.get();
  P.descs = pages->d_descs.get();
  P.time_page_of = pages->d_time_page_of.get();
  P.work_page = s->d_work_page.get();
  P.work_slot = s->d_work_slot.get();
  P.work_qcol = s->d_work_qcol.get();
  P.region_start = s->d_region.get();
  P.region_fill = s->d_bucket.get();
  P.cols = s->d_cols.get();
  P.state = slide ? s->d_pane_state.get() : s->d_state.get();
  P.task_counter = reinterpret_cast<uint32_t *>(s->d_aux.get());
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
  P.edges = s->d_edges.get();
  P.n_buckets = E.on ? E.n : s->n_panes;  // (a labelled scan: its edge buckets; n_panes = its output buckets)
  P.cell_buckets = E.labelled ? q->n_buckets : 0;
  P.group_by_series = q->group_by_series;
  P.n_cells = L.n_groups * s->n_panes;
  P.slot_group = s->d_slot_group.get();
  P.slot_bits = slot_bits;
  P.slot_max = slot_bits ? (uint32_t)((1ull << slot_bits) - 1) : 0;
  P.rel_base = rel_base;
  P.use_smem = lay.use_smem;
  P.smem_words = lay.smem_words;
  P.n_cols = q->n_columns;
  P.row_keep = s->d_row_keep.get();
  P.keep_off = pages->d_keep_off.get();
  P.skip_off = pages->d_skip_off.get();
  P.page_narrow = pages->d_narrow.get();
  P.skip = pages->d_skip.get();
  P.has_tomb = pages->tomb.n_ranges ? 1u : 0u;
  P.tomb_keys = pages->tomb.keys.get();
  P.tomb_off = pages->tomb.off.get();
  P.tomb_ranges = pages->tomb.ranges.get();
  P.n_tomb_keys = pages->tomb.n_keys;
  P.n_tomb_global = pages->tomb.n_global;
  s->tomb_epoch = pages->tomb_epoch;
  plan_grids(ctx, pages, q, has_sel, P.edges != nullptr, P.smem_words, P.has_tomb, s->grid, s->occ, P.bin_parts, P.bin_part_rows);
  if (s->n_m2) {  // pass 2: the same scan over the M2 columns' regions, with its own fills, task counters and tables
    ScanParams &P2 = s->params2;
    P2 = P;
    P2.cols = s->d_cols2.get();
    P2.region_fill = s->d_fill2.get();
    P2.task_counter = s->d_fill2.get() + N_BINS * q->n_columns * WL_SUB;
    P2.use_smem = lay.use_smem2;
    P2.smem_words = lay.smem_words2;
  }
  s->chunk_epoch = pages->chunk_epoch;
  if (pages->overlap.merge_rows && (st = prepare_merge(ctx, pages, q, s, &h2d)) != TSKV_OK) {
    delete s;
    return st;
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

tskv_status tskvgpu_scan_prepare_edges(tskv_ctx *ctx, const tskv_pages *pages, const tskv_query *q, const int64_t *edges,
                                       const uint32_t *group_ids, uint32_t n_groups, tskv_scan **out_scan) {
  return prepare_scan(ctx, pages, q, 0, TagGroups{group_ids != nullptr, group_ids, n_groups}, out_scan, plain_edges(q, edges));
}

tskv_status tskvgpu_scan_prepare_labels(tskv_ctx *ctx, const tskv_pages *pages, const tskv_query *q, const int64_t *edges,
                                        uint32_t n_edge, const uint32_t *labels, const uint32_t *group_ids, uint32_t n_groups,
                                        tskv_scan **out_scan) {
  return prepare_scan(ctx, pages, q, 0, TagGroups{group_ids != nullptr, group_ids, n_groups}, out_scan,
                      BucketEdges{true, edges, n_edge, true, labels});
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
  if (!capturing) cudaEventRecord(s->ev0.get(), ctx->stream.get());
  unsigned long long *aux = s->d_aux.get();
  uint64_t launches = 0;
  const SeriesIndex series{pages->d_series_sorted.get(), pages->d_rank_of.get(), (uint32_t)pages->series.size(), pages->series_min,
                           pages->series_span};
  {  // state identities + the pass's scratch (task counters / status / counters, work-list bucket fills): one launch
    const uint32_t init_blocks = (uint32_t)std::min<uint64_t>((s->kern_sl.total + 255) / 256, 4096);
    k_init_state<<<std::max(1u, init_blocks), 256, 0, ctx->stream.get()>>>(s->params.state, s->kern_sl, aux, AUX_WORDS, s->d_bucket.get(),
                                                                   N_BINS * s->n_cols * WL_SUB);
    launches++;
  }
  // slot of every column group: the row filter and the merge pass need it per GROUP; the work list finds a selected
  // series' groups itself
  const bool need_cg_slot = s->preds.n || (s->merge.n_rows && s->n_merge_pages);
  if (pages->n_cg && need_cg_slot) {
    if (s->d_rank_slot) {
      CU_TRY(ctx, cudaMemsetAsync(s->d_rank_slot.get(), 0xff, pages->series.size() * 4, ctx->stream.get()));
      if (s->n_series_sel) {
        k_select_ids<<<(s->n_series_sel + 255) / 256, 256, 0, ctx->stream.get()>>>(series, s->d_series.get(), s->n_series_sel,
                                                                         s->d_rank_slot.get());
        launches++;
      }
    }
    k_select_cg<<<(pages->n_cg + 255) / 256, 256, 0, ctx->stream.get()>>>(pages->n_cg, s->d_rank_slot.get(), pages->d_cg_series_rank.get(), s->d_cg_slot.get());
    launches++;
  }
  if (s->preds.n && pages->n_cg) {  // row filter: keep bits of every selected column group (host-resident pages: read in place)
    k_row_filter<<<(pages->n_cg + 127) / 128, 128, 0, ctx->stream.get()>>>(pages->h_mapped ? pages->h_mapped : pages->d_arena.get(), pages->d_descs.get(),
                                                                     pages->n_descs, pages->d_cg_time_page.get(), pages->n_cg, s->d_cg_slot.get(),
                                                                     s->preds, pages->d_keep_off.get(), s->d_row_keep.get(), s->d_status, s->d_err_page);
    launches++;
  }
  if (n_items) {
    WorkListArgs A{};
    A.descs = pages->d_descs.get();
    A.n_descs = pages->n_descs;
    A.cg_time_page = pages->d_cg_time_page.get();
    A.n_cg = pages->n_cg;
    A.rank_cg_start = pages->d_rank_cg_start.get();
    A.rank_cg = pages->d_rank_cg.get();
    A.page_bin = pages->d_page_bin.get();
    // narrow pages apart only where a bin holds both kinds (NARROW_SOME kernels choose per chunk)
    A.page_narrow = s->split_narrow ? pages->d_narrow.get() : nullptr;
    A.series = series;
    A.series_ids = s->d_series.get();
    A.n_sel = s->d_series ? s->n_series_sel : (uint32_t)pages->series.size();
    A.split_log2 = s->walk_split_log2;
    A.walk = s->d_walk.get();
    A.cols = s->d_cols.get();
    A.n_cols = s->n_cols;
    A.cg_bounds = s->prune.n ? pages->d_cg_bounds.get() : nullptr;
    A.prune = s->prune;
    A.cg_merge = pages->overlap.d_cg_merge.get();
    A.page_stats = s->preds.n ? pages->d_page_stats.get() : nullptr;
    A.preds = s->preds;
    A.region_start = s->d_region.get();
    A.bucket_fill = s->d_bucket.get();
    A.work_page = s->d_work_page.get();
    A.work_slot = s->d_work_slot.get();
    A.work_qcol = s->d_work_qcol.get();
    A.counters = s->d_counters;
    A.status = s->d_status;
    const uint32_t wblocks = std::max(1u, (uint32_t)((((uint64_t)A.n_sel << A.split_log2) + WL_THREADS - 1) / WL_THREADS));
    if (A.n_sel) {
      k_worklist<<<wblocks, WL_THREADS, 2 * N_BINS * s->n_cols * WL_SUB * 4, ctx->stream.get()>>>(A);
      launches++;
    }
  }
  if (s->merge.n_rows && s->n_merge_pages) {  // overlapping chunks: decode the query's columns, merge + aggregate per row
    CU_TRY(ctx, cudaMemsetAsync(s->d_mvalid.get(), 0, (size_t)s->n_cols * s->merge.bm_words * 4, ctx->stream.get()));
    const uint32_t dblocks = (uint32_t)(((uint64_t)s->n_merge_pages * 32 + DECODE_THREADS - 1) / DECODE_THREADS);
    k_decode_warp<<<dblocks, DECODE_THREADS, 0, ctx->stream.get()>>>(pages->h_mapped ? pages->h_mapped : pages->d_arena.get(), pages->d_descs.get(), 0, s->d_mpage.get(),
                                                              s->n_merge_pages, s->d_mrow_off.get(), s->d_mbm_off.get(), s->d_mvals.get(),
                                                              reinterpret_cast<uint8_t *>(s->d_mvalid.get()), s->d_status, s->d_err_page, s->d_stats);
    const uint32_t mblocks = (uint32_t)((s->merge.n_rows + 127) / 128);
    k_merge_chunks<false><<<mblocks, 128, 0, ctx->stream.get()>>>(s->params, s->merge);
    launches += 2;
  }
  cudaEvent_t ev_fork = capturing ? s->ev_cfork.get() : s->ev_bin[0].get();
  cudaEventRecord(ev_fork, ctx->stream.get());  // fork
  // Host-resident pages: one bin's gather already saturates PCIe, so the gathers are chained largest bin first
  // (an event per bin); each bin's CRC check and scan then overlap the next bins' transfers and only the smallest
  // bin's tail is exposed after the last byte has arrived.
  int order[N_BINS];
  for (int b = 0; b < N_BINS; b++) order[b] = b;
  if (pages->h_mapped)
    std::stable_sort(order, order + N_BINS, [&](int a, int b) { return pages->h_bin_bytes[a] > pages->h_bin_bytes[b]; });
  else
    std::stable_sort(order, order + N_BINS, [&](int a, int b) { return chunk_cost(a) > chunk_cost(b); });
  int prev_gather = -1;
  for (int oi = 0; oi < N_BINS; oi++) {
    const int b = order[oi];
    if (!s->grid[b]) continue;
    cudaStreamWaitEvent(ctx->bin_stream[b].get(), ev_fork, 0);
    int bin = b;
    const uint32_t n_bin = pages->h_bin_pages[b];
    if (pages->h_mapped) {
      if (prev_gather >= 0) cudaStreamWaitEvent(ctx->bin_stream[b].get(), s->ev_gather[prev_gather].get(), 0);
      uint32_t gblocks = std::max(1u, std::min<uint32_t>((uint32_t)ctx->sm_count * 4, (n_bin + 7) / 8));
      k_gather_pages<<<gblocks, 256, 0, ctx->bin_stream[b].get()>>>(pages->h_mapped, pages->d_arena.get(), pages->d_descs.get(),
                                                              pages->d_time_page_of.get(), s->d_work_page.get(), s->d_work_qcol.get(),
                                                              s->d_region.get(), s->d_bucket.get(), s->n_cols * WL_SUB, bin);
      launches++;
      cudaEventRecord(s->ev_gather[b].get(), ctx->bin_stream[b].get());
      prev_gather = b;
    }
    if (pages->verify_on_read) {  // Page::crc_validation on every read (tsm/reader.rs:259), also for pages resident in HBM
      // In front of the bin's fused kernel (HBM-resident pages) / after the bin's transfer, under the next bin's
      // (host-resident pages). Beside the fused kernels on a stream of its own the check was slower (H100, C4: 1.84-2.03
      // ms per scan with 1-8 CRC blocks per SM against 1.39 ms in line): it needs the whole machine's lanes to hide its
      // dependent table lookups. A mismatch is reported in its own status slot and outranks whatever the decoders made of
      // the corrupt page.
      uint32_t gblocks = std::max(1u, std::min<uint32_t>((uint32_t)ctx->sm_count * 4, (n_bin + 7) / 8));
      k_verify_crc<<<gblocks, 256, 0, ctx->bin_stream[b].get()>>>(pages->d_arena.get(), pages->d_descs.get(), pages->d_time_page_of.get(),
                                                            s->d_work_page.get(), s->d_work_qcol.get(), s->d_region.get(), s->d_bucket.get(),
                                                            s->n_cols * WL_SUB, bin,
                                                            pages->d_crc_tables.get(), s->d_crc_status, s->d_crc_err_page);
      launches++;
    }
    if (!capturing) cudaEventRecord(s->ev_bin_start[b].get(), ctx->bin_stream[b].get());
    const int sb = serial_bin_of(b);
    void *args[] = {(void *)&s->params, (void *)&bin};
    const bool edges = s->params.edges != nullptr;
    const void *fn = (const void *)(s->has_sel ? scan_kernel_for<true>(sb, edges) : scan_kernel_for<false>(sb, edges, pages->h_bin_narrow[b]));
    CU_TRY(ctx, cudaLaunchKernel(fn, dim3(s->grid[b]), dim3(SCAN_THREADS), args, serial_smem_bytes(sb, s->params.smem_words, s->params.has_tomb),
                                 ctx->bin_stream[b].get()));
    cudaEvent_t ev_done = capturing ? s->ev_cjoin[b].get() : s->ev_bin_done[b].get();
    cudaEventRecord(ev_done, ctx->bin_stream[b].get());
    cudaStreamWaitEvent(ctx->stream.get(), ev_done, 0);  // join
    launches++;
  }
  if (!capturing && !s->n_m2 && !s->n_pairs && !s->n_medians && !s->n_increases) cudaEventRecord(s->ev_bin[N_BINS].get(), ctx->stream.get());
  if (s->n_combine) {  // sliding windows: every window folds its panes (it writes every array the kernels fill)
    const uint32_t bx = (uint32_t)std::min<uint64_t>((s->layout.n_cells + 255) / 256, 1024);
    k_window_combine<<<dim3(std::max(1u, bx), s->n_combine), 256, 0, ctx->stream.get()>>>(
        s->d_pane_state.get(), s->d_state.get(), s->d_combine.get(), (uint32_t)s->layout.n_groups, s->n_windows, s->n_panes, s->win_k);
    launches++;
  }
  if (s->has_sel || s->n_means) {
    uint64_t work = std::max(std::max(s->sl.first_cells, s->sl.last_cells), s->n_means ? s->layout.n_cells : 0);
    uint32_t b = (uint32_t)std::min<uint64_t>((work + 255) / 256, 4096);
    k_export_pairs<<<std::max(1u, b), 256, 0, ctx->stream.get()>>>(s->d_state.get(), s->sl, s->d_means.get(), s->n_means, s->layout.n_cells);
    launches++;
  }
  if (s->n_m2) {  // TSKV_AGG_M2, pass 2: every cell's shift (pass-1 mean), then the M2 columns' rows once more
    const uint32_t nb = N_BINS * s->n_cols * WL_SUB;
    const uint32_t bx = (uint32_t)std::min<uint64_t>((s->layout.n_cells + 255) / 256, 1024);
    k_m2_prep<<<dim3(std::max(1u, bx), s->n_m2), 256, 0, ctx->stream.get()>>>(s->d_state.get(), s->d_m2.get(), s->layout.n_cells,
                                                                          s->d_bucket.get(), s->d_fill2.get(), nb, s->d_cols2.get(),
                                                                          s->n_cols, s->params2.task_counter);
    launches++;
    if (s->merge.n_rows && s->n_merge_pages) {
      k_merge_chunks<true><<<(uint32_t)((s->merge.n_rows + 127) / 128), 128, 0, ctx->stream.get()>>>(s->params2, s->merge);
      launches++;
    }
    cudaEventRecord(s->ev_m2_fork.get(), ctx->stream.get());
    const bool edges = s->params.edges != nullptr;
    for (int b = 0; b < N_BINS; b++) {
      if (!s->grid[b] || !s->m2_bin[b]) continue;
      cudaStreamWaitEvent(ctx->bin_stream[b].get(), s->ev_m2_fork.get(), 0);
      int bin = b;
      const int sb = serial_bin_of(b);
      void *args[] = {(void *)&s->params2, (void *)&bin};
      CU_TRY(ctx, cudaLaunchKernel((const void *)m2_kernel_for(sb, edges), dim3(s->grid[b]), dim3(SCAN_THREADS), args,
                                   serial_smem_bytes(sb, s->params2.smem_words, s->params2.has_tomb), ctx->bin_stream[b].get()));
      cudaEventRecord(s->ev_m2_join[b].get(), ctx->bin_stream[b].get());
      cudaStreamWaitEvent(ctx->stream.get(), s->ev_m2_join[b].get(), 0);
      launches++;
    }
    if (!capturing && !s->n_pairs && !s->n_medians && !s->n_increases) cudaEventRecord(s->ev_bin[N_BINS].get(), ctx->stream.get());  // (the fused time includes pass 2)
  }
  if (s->n_pairs) {  // column pairs: pass 1 (n, sums, extremes), the shifts, pass 2 (co-moments); overlap merge rows first
    const bool edges = s->params.edges != nullptr;
    const uint32_t bx = (uint32_t)std::min<uint64_t>((s->layout.n_cells + 255) / 256, 1024);
    const uint32_t px = (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>(((uint64_t)pages->n_descs + 127) / 128, (uint64_t)ctx->sm_count * 16));
    const bool merge = s->merge.n_rows && s->n_merge_pages;
    for (int pass = 0; pass < 2; pass++) {
      if (pass == 1) {
        k_pair_prep<<<dim3(std::max(1u, bx), s->n_pairs), 256, 0, ctx->stream.get()>>>(s->d_state.get(), s->d_pairs.get(), s->layout.n_cells);
        launches++;
      }
      if (merge) {
        const uint32_t mb = (uint32_t)((s->merge.n_rows + 127) / 128);
        if (pass) k_merge_pairs_rows<true><<<mb, 128, 0, ctx->stream.get()>>>(s->params, s->merge, s->d_pairs.get(), s->n_pairs);
        else k_merge_pairs_rows<false><<<mb, 128, 0, ctx->stream.get()>>>(s->params, s->merge, s->d_pairs.get(), s->n_pairs);
        launches++;
      }
      const void *fn = pass ? (edges ? (const void *)k_scan_pair<true, true> : (const void *)k_scan_pair<true, false>)
                            : (edges ? (const void *)k_scan_pair<false, true> : (const void *)k_scan_pair<false, false>);
      const PairCol *pp = s->d_pairs.get();
      uint64_t nd = pages->n_descs;
      void *args[] = {(void *)&s->params, (void *)&pp, (void *)&nd};
      CU_TRY(ctx, cudaLaunchKernel(fn, dim3(px, s->n_pairs), dim3(128), args, 0, ctx->stream.get()));
      launches++;
    }
    if (!capturing && !s->n_medians && !s->n_increases) cudaEventRecord(s->ev_bin[N_BINS].get(), ctx->stream.get());  // (the fused time includes the pair passes)
  }
  if (s->n_medians) {  // medians: the targets from pass 1, then MEDIAN_PASSES fixed selection passes (merged rows first)
    const bool edges = s->params.edges != nullptr;
    const uint64_t n_cells = s->layout.n_cells;
    const uint32_t bx = (uint32_t)std::min<uint64_t>((n_cells + 255) / 256, 1024);
    const uint32_t wx = (uint32_t)std::min<uint64_t>((n_cells + 7) / 8, 4096);  // k_median_step: a warp per cell
    const uint32_t px = (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>(((uint64_t)pages->n_descs + 127) / 128, (uint64_t)ctx->sm_count * 16));
    const bool merge = s->merge.n_rows && s->n_merge_pages;
    CU_TRY(ctx, cudaMemsetAsync(s->med.unresolved, 0, sizeof(unsigned long long), ctx->stream.get()));
    k_median_prep<<<dim3(std::max(1u, bx), s->n_medians), 256, 0, ctx->stream.get()>>>(s->d_state.get(), s->d_medians.get(), s->med, n_cells);
    launches++;
    const void *fn = edges ? (const void *)k_scan_median<true> : (const void *)k_scan_median<false>;
    const MedianCol *mp = s->d_medians.get();
    void *args[] = {(void *)&s->params, (void *)&mp, (void *)&s->med};
    for (int pass = 0; pass < MEDIAN_PASSES; pass++) {
      if (merge) {
        k_merge_median_rows<<<(uint32_t)((s->merge.n_rows + 127) / 128), 128, 0, ctx->stream.get()>>>(s->params, s->merge, mp, s->n_medians, s->med);
        launches++;
      }
      CU_TRY(ctx, cudaLaunchKernel(fn, dim3(px, s->n_medians), dim3(128), args, 0, ctx->stream.get()));
      k_median_step<<<dim3(std::max(1u, wx), s->n_medians), 256, 0, ctx->stream.get()>>>(mp, s->med, n_cells);
      launches += 2;
    }
    if (!capturing && !s->n_increases) cudaEventRecord(s->ev_bin[N_BINS].get(), ctx->stream.get());  // (the fused time includes the selection passes)
  }
  if (s->n_increases) {  // increases: the pages' pairs and records and the merged rows' records, then the boundaries
    const bool edges = s->params.edges != nullptr;
    const uint64_t n = (uint64_t)s->inc.n_rec * s->n_increases;
    const uint32_t nb = (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>((n + 255) / 256, 4096));
    const uint32_t px = (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>(((uint64_t)pages->n_descs + 127) / 128, (uint64_t)ctx->sm_count * 16));
    uint64_t *keys = s->d_inc_keys.get();
    uint32_t *idx = s->d_inc_idx.get();
    const IncreaseCol *ip = s->d_increases.get();
    k_increase_init<<<nb, 256, 0, ctx->stream.get()>>>(s->inc, n, idx);
    const void *fn = edges ? (const void *)k_scan_increase<true> : (const void *)k_scan_increase<false>;
    void *args[] = {(void *)&s->params, (void *)&ip, (void *)&s->inc};
    CU_TRY(ctx, cudaLaunchKernel(fn, dim3(px, s->n_increases), dim3(128), args, 0, ctx->stream.get()));
    launches += 2;
    if (s->merge.n_rows && s->n_merge_pages) {
      k_merge_increase<<<dim3((uint32_t)((s->merge.n_rows + 127) / 128), s->n_increases), 128, 0, ctx->stream.get()>>>(
          s->params, s->merge, ip, s->inc, (uint32_t)(s->inc.n_rec - s->n_inc_merge_rows));
      launches++;
    }
    // records by first time, then (stably) by (increase, slot): keys [slot | time | time sorted | slot in time order |
    // slot sorted], indices [identity | time order | final order]; each sort reads only its keys' bits (alloc_scan)
    size_t tmp = s->inc_tmp_bytes;
    CU_TRY(ctx, cub::DeviceRadixSort::SortPairs(s->d_inc_tmp.get(), tmp, keys + n, keys + 2 * n, idx, idx + n, (int)n, 0,
                                                s->inc_time_sort_bits, ctx->stream.get()));
    k_increase_gather<<<nb, 256, 0, ctx->stream.get()>>>(keys, idx + n, n, keys + 3 * n);
    tmp = s->inc_tmp_bytes;
    CU_TRY(ctx, cub::DeviceRadixSort::SortPairs(s->d_inc_tmp.get(), tmp, keys + 3 * n, keys + 4 * n, idx + n, idx + 2 * n, (int)n, 0,
                                                s->inc_slot_sort_bits, ctx->stream.get()));
    k_increase_stitch<<<nb, 256, 0, ctx->stream.get()>>>(s->d_state.get(), ip, s->inc, keys + 4 * n, idx + 2 * n, n);
    launches += 4;  // (a sort counts as one launch)
    if (!capturing) cudaEventRecord(s->ev_bin[N_BINS].get(), ctx->stream.get());  // (the fused time includes the increase kernels)
  }
  if (!capturing) cudaEventRecord(s->ev1.get(), ctx->stream.get());
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
  unsigned long long aux[AUX_COUNTERS + N_COUNTERS - AUX_STATS] = {0};  // the stats, then the reader counters
  CU_TRY(ctx, cudaMemcpy(aux, s->d_stats, sizeof(aux), cudaMemcpyDeviceToHost));
  const unsigned long long *ctr = aux + (AUX_COUNTERS - AUX_STATS);
  ctx->counters.pruned_page_count = ctr[CTR_PRUNED];
  float ms = 0;
  cudaEventElapsedTime(&ms, s->ev0.get(), s->ev1.get());
  ctx->counters.elapsed_scan_ms = ms;
  ctx->counters.points_decoded = aux[0];
  ctx->counters.rows_in_range = aux[1];
  ctx->counters.page_read_count = ctr[CTR_PAGES] + s->merge_read_pages;
  ctx->counters.page_read_bytes = ctr[CTR_BYTES] + s->merge_page_bytes;
  float fused = 0;
  cudaEventElapsedTime(&fused, s->ev_bin[0].get(), s->ev_bin[N_BINS].get());
  ctx->counters.elapsed_fused_ms = fused;
  ctx->counters.dominant_kernel_ms = 0;
  ctx->counters.dominant_kernel_bytes = 0;
  ctx->counters.dominant_kernel_bin = 0;
  if (getenv("TSKV_DEBUG_BINS")) {  // (events of the un-captured pass: meaningful with TSKV_NO_GRAPH=1)
    float pro = 0, epi = 0;
    cudaEventElapsedTime(&pro, s->ev0.get(), s->ev_bin[0].get());
    cudaEventElapsedTime(&epi, s->ev_bin[N_BINS].get(), s->ev1.get());
    fprintf(stderr, "[tskv] prologue (select, work list, init%s) %.3f ms, fused %.3f ms, epilogue %.3f ms\n",
            s->merge.n_rows ? ", merge pass" : "", pro, fused, epi);
  }
  for (int b = 0; b < N_BINS; b++) {
    if (!s->grid[b]) continue;
    float t = 0;
    cudaEventElapsedTime(&t, s->ev_bin_start[b].get(), s->ev_bin_done[b].get());
    if (getenv("TSKV_DEBUG_BINS")) {
      float t0 = 0;
      cudaEventElapsedTime(&t0, s->ev_bin[0].get(), s->ev_bin_start[b].get());
      fprintf(stderr, "[tskv] bin %d grid %d, %d CTAs/SM: start +%.3f ms, run %.3f ms, %llu bytes\n", b,
              s->grid[b], s->occ[b], t0, t, ctr[CTR_BIN_BYTES + b]);
    }
    if (t > ctx->counters.dominant_kernel_ms) {
      ctx->counters.dominant_kernel_ms = t;
      ctx->counters.dominant_kernel_bytes = ctr[CTR_BIN_BYTES + b];
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
      s->ev_cfork = new_event(cudaEventDisableTiming);
      for (int b = 0; b < N_BINS; b++) s->ev_cjoin[b] = new_event(cudaEventDisableTiming);
    }
    bool ok = cudaStreamBeginCapture(ctx->stream.get(), cudaStreamCaptureModeThreadLocal) == cudaSuccess;
    if (ok) {
      const tskv_status st = enqueue_scan(ctx, s, true);  // the bin streams join the capture through the fork event
      const cudaError_t e = cudaStreamEndCapture(ctx->stream.get(), &graph);
      cudaGraphExec_t exec = nullptr;
      ok = st == TSKV_OK && e == cudaSuccess && graph && cudaGraphInstantiate(&exec, graph, 0) == cudaSuccess;
      s->graph_exec.reset(ok ? exec : nullptr);
      if (graph) cudaGraphDestroy(graph);
    }
    if (!ok) {  // anything the capture did not like: replay the pass call by call, as before
      if (getenv("TSKV_DEBUG_BINS")) fprintf(stderr, "[tskv] graph capture failed (%s): direct launches\n", cudaGetErrorString(cudaGetLastError()));
      cudaGetLastError();
      s->graph_failed = true;
      return enqueue_scan(ctx, s);
    }
  }
  CU_TRY(ctx, cudaGraphLaunch(s->graph_exec.get(), ctx->stream.get()));
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

tskv_status tskvgpu_scan_work_list(tskv_ctx *ctx, tskv_scan *s, uint32_t *n_buckets, uint32_t *n_items, uint32_t *region_start,
                                   uint32_t *fill, uint32_t *work_page, uint32_t *work_slot, uint8_t *work_qcol, uint8_t *page_bin,
                                   uint8_t *page_narrow) {
  if (!ctx || !s || !n_buckets || !n_items) return TSKV_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(ctx->mu);
  ctx->set_error("");
  CU_TRY(ctx, cudaSetDevice(ctx->device));
  const tskv_pages *pages = s->pages;
  const uint32_t nb = N_BINS * s->n_cols * WL_SUB;
  std::vector<uint32_t> start(nb + 1);
  CU_TRY(ctx, cudaStreamSynchronize(ctx->stream.get()));
  CU_TRY(ctx, cudaMemcpy(start.data(), s->d_region.get(), start.size() * 4, cudaMemcpyDeviceToHost));
  *n_buckets = nb;
  *n_items = start[nb];
  if (region_start) std::copy(start.begin(), start.end(), region_start);
  if (fill) CU_TRY(ctx, cudaMemcpy(fill, s->d_bucket.get(), (size_t)nb * 4, cudaMemcpyDeviceToHost));
  if (work_page && start[nb]) CU_TRY(ctx, cudaMemcpy(work_page, s->d_work_page.get(), (size_t)start[nb] * 4, cudaMemcpyDeviceToHost));
  if (work_slot && start[nb]) CU_TRY(ctx, cudaMemcpy(work_slot, s->d_work_slot.get(), (size_t)start[nb] * 4, cudaMemcpyDeviceToHost));
  if (work_qcol && start[nb]) CU_TRY(ctx, cudaMemcpy(work_qcol, s->d_work_qcol.get(), start[nb], cudaMemcpyDeviceToHost));
  if (page_bin && pages->n_descs) CU_TRY(ctx, cudaMemcpy(page_bin, pages->d_page_bin.get(), pages->n_descs, cudaMemcpyDeviceToHost));
  if (page_narrow && pages->n_descs) {
    if (s->split_narrow) CU_TRY(ctx, cudaMemcpy(page_narrow, pages->d_narrow.get(), pages->n_descs, cudaMemcpyDeviceToHost));
    else std::memset(page_narrow, 0, pages->n_descs);
  }
  return TSKV_OK;
}

// Medians keep no mergeable partial state: the exchange calls refuse a scan with medians.
static tskv_status refuse_medians(tskv_ctx *ctx, const tskv_scan *s, const char *call) {
  if (!s->n_medians) return TSKV_OK;
  std::lock_guard<std::mutex> lock(ctx->mu);
  ctx->set_error(std::string(call) + ": a scan with medians has no mergeable partial state");
  return TSKV_ERR_UNSUPPORTED;
}

tskv_status tskvgpu_scan_partials(tskv_ctx *ctx, tskv_scan *s, tskv_partials_view *out) {
  if (!ctx || !s || !out) return TSKV_ERR_INVALID_ARG;
  if (tskv_status st = refuse_medians(ctx, s, "scan_partials")) return st;
  if (s->n_m2 || s->n_pairs) {
    std::lock_guard<std::mutex> lock(ctx->mu);
    ctx->set_error("scan_partials: second moments (TSKV_AGG_M2, column pairs) do not all-reduce element-wise; use tskvgpu_scan_exchange");
    return TSKV_ERR_UNSUPPORTED;
  }
  const StateLayout &L = s->sl;
  uint64_t base = (uint64_t)(uintptr_t)s->d_state.get();
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

// The M2 columns of gathered partials: Chan's merge of every rank's (count, sum, M2) (k_merge_m2).
// (and the column pairs: Chan's merge of every rank's n, means and co-moments, k_merge_pairs)
static void merge_m2(tskv_ctx *ctx, tskv_scan *s, const uint64_t *gathered, uint32_t n_ranks, uint64_t words) {
  const uint32_t bx = (uint32_t)std::min<uint64_t>((s->layout.n_cells + 255) / 256, 1024);
  if (s->n_m2)
    k_merge_m2<<<dim3(std::max(1u, bx), s->n_m2), 256, 0, ctx->stream.get()>>>(s->d_state.get(), s->d_m2.get(), s->layout.n_cells, gathered,
                                                                           n_ranks, words);
  if (s->n_pairs)
    k_merge_pairs<<<dim3(std::max(1u, bx), s->n_pairs), 256, 0, ctx->stream.get()>>>(s->d_state.get(), s->d_pairs.get(), s->layout.n_cells,
                                                                                 gathered, n_ranks, words);
}

tskv_status tskvgpu_scan_exchange_view(tskv_ctx *ctx, tskv_scan *s, uint64_t *out_dptr, uint64_t *out_words) {
  if (!ctx || !s || !out_dptr || !out_words) return TSKV_ERR_INVALID_ARG;
  if (tskv_status st = refuse_medians(ctx, s, "scan_exchange_view")) return st;
  *out_dptr = (uint64_t)(uintptr_t)s->d_state.get();
  *out_words = s->sl.selval_off + s->sl.selval_len + s->m2_words + s->pair_words;  // sum_i64 | sum_f64 | min+first keys | max+last keys | values | M2 | pairs
  return TSKV_OK;
}

tskv_status tskvgpu_scan_merge_gathered(tskv_ctx *ctx, tskv_scan *s, uint64_t gathered_dptr, uint32_t n_ranks) {
  if (!ctx || !s || !gathered_dptr || n_ranks == 0) return TSKV_ERR_INVALID_ARG;
  if (tskv_status st = refuse_medians(ctx, s, "scan_merge_gathered")) return st;
  std::lock_guard<std::mutex> lock(ctx->mu);
  cudaSetDevice(ctx->device);
  const uint64_t words = s->sl.selval_off + s->sl.selval_len + s->m2_words + s->pair_words;
  uint32_t blocks = (uint32_t)std::min<uint64_t>((words + 255) / 256, 2048);
  k_merge_gathered<<<std::max(1u, blocks), 256, 0, ctx->stream.get()>>>(s->d_state.get(), s->sl, reinterpret_cast<const uint64_t *>((uintptr_t)gathered_dptr),
                                                                   n_ranks, words);
  merge_m2(ctx, s, reinterpret_cast<const uint64_t *>((uintptr_t)gathered_dptr), n_ranks, words);
  CU_TRY(ctx, cudaGetLastError());
  return TSKV_OK;
}

tskv_status tskvgpu_scan_exchange(tskv_ctx *ctx, tskv_scan *s) {
  if (!ctx || !s) return TSKV_ERR_INVALID_ARG;
  if (tskv_status st = refuse_medians(ctx, s, "scan_exchange")) return st;
  std::lock_guard<std::mutex> lock(ctx->mu);
  cudaSetDevice(ctx->device);
  if (!ctx->comm) {
    ctx->set_error("tskvgpu_scan_exchange: no communicator (tskvgpu_comm_init)");
    return TSKV_ERR_NCCL;
  }
  const NcclApi &N = nccl_api();
  const uint64_t words = s->sl.selval_off + s->sl.selval_len + s->m2_words + s->pair_words;  // sum_i64 | sum_f64 | min+first keys | max+last keys | values | M2
  if (!s->d_gathered) CU_TRY(ctx, stream_alloc(s->d_gathered, (size_t)ctx->n_ranks * words, ctx->stream.get()));
  const ncclResult_t r = N.AllGather(s->d_state.get(), s->d_gathered.get(), words, ncclUint64, ctx->comm, ctx->stream.get());
  if (r != ncclSuccess) {
    ctx->set_error(std::string("ncclAllGather: ") + N.GetErrorString(r));
    return TSKV_ERR_NCCL;
  }
  uint32_t blocks = (uint32_t)std::min<uint64_t>((words + 255) / 256, 2048);
  k_merge_gathered<<<std::max(1u, blocks), 256, 0, ctx->stream.get()>>>(s->d_state.get(), s->sl, s->d_gathered.get(), (uint32_t)ctx->n_ranks, words);
  merge_m2(ctx, s, s->d_gathered.get(), (uint32_t)ctx->n_ranks, words);
  CU_TRY(ctx, cudaGetLastError());
  return TSKV_OK;
}

tskv_status tskvgpu_scan_snapshot_keys(tskv_ctx *ctx, tskv_scan *s) {
  if (!ctx || !s) return TSKV_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(ctx->mu);
  cudaSetDevice(ctx->device);
  if (s->has_sel) {
    k_snapshot_keys<<<256, 256, 0, ctx->stream.get()>>>(s->d_state.get(), s->sl);
    CU_TRY(ctx, cudaGetLastError());
  }
  return TSKV_OK;
}

tskv_status tskvgpu_scan_mask_values(tskv_ctx *ctx, tskv_scan *s) {
  if (!ctx || !s) return TSKV_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(ctx->mu);
  cudaSetDevice(ctx->device);
  if (s->has_sel) {
    k_mask_values<<<256, 256, 0, ctx->stream.get()>>>(s->d_state.get(), s->sl);
    CU_TRY(ctx, cudaGetLastError());
  }
  return TSKV_OK;
}

static tskv_status finalize_device(tskv_ctx *ctx, tskv_scan *s) {
  const tskv_output_layout &L = s->layout;
  if (s->n_out) {
    dim3 grid((uint32_t)((L.n_cells + 255) / 256), s->n_out);
    k_finalize<<<grid, 256, 0, ctx->stream.get()>>>(s->d_state.get(), s->d_outs.get(), s->n_out, L.n_cells, L.bitmap_stride, s->d_values.get(),
                                              s->d_validity.get());
  }
  if (s->n_pairs)
    k_finalize_pairs<<<dim3((uint32_t)((L.n_cells + 255) / 256), 4 * s->n_pairs), 256, 0, ctx->stream.get()>>>(
        s->d_state.get(), s->d_pairs.get(), s->n_out, L.n_cells, L.bitmap_stride, s->d_values.get(), s->d_validity.get());
  if (s->n_medians)
    k_finalize_medians<<<dim3((uint32_t)((L.n_cells + 255) / 256), s->n_medians), 256, 0, ctx->stream.get()>>>(
        s->d_state.get(), s->d_medians.get(), s->med, s->n_out + 4 * s->n_pairs, L.n_cells, L.bitmap_stride, s->d_values.get(),
        s->d_validity.get());
  if (s->n_increases)
    k_finalize_increases<<<dim3((uint32_t)((L.n_cells + 255) / 256), s->n_increases), 256, 0, ctx->stream.get()>>>(
        s->d_state.get(), s->d_increases.get(), s->n_out + 4 * s->n_pairs + s->n_medians, L.n_cells, L.bitmap_stride, s->d_values.get(),
        s->d_validity.get());
  CU_TRY(ctx, cudaGetLastError());
  return TSKV_OK;
}

tskv_status tskvgpu_scan_finalize(tskv_ctx *ctx, tskv_scan *s, uint64_t *out_values, uint8_t *out_validity) {
  if (!ctx || !s || !out_values || !out_validity) return TSKV_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(ctx->mu);
  cudaSetDevice(ctx->device);
  tskv_status st = finalize_device(ctx, s);
  if (st != TSKV_OK) return st;
  CU_TRY(ctx, cudaMemcpyAsync(out_values, s->d_values.get(), s->layout.values_bytes, cudaMemcpyDeviceToHost, ctx->stream.get()));
  CU_TRY(ctx, cudaMemcpyAsync(out_validity, s->d_validity.get(), s->layout.validity_bytes, cudaMemcpyDeviceToHost, ctx->stream.get()));
  CU_TRY(ctx, cudaStreamSynchronize(ctx->stream.get()));
  return TSKV_OK;
}

tskv_status tskvgpu_scan_finalize_device(tskv_ctx *ctx, tskv_scan *s, uint64_t *out_values_dptr,
                                         uint64_t *out_validity_dptr) {
  if (!ctx || !s) return TSKV_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(ctx->mu);
  cudaSetDevice(ctx->device);
  tskv_status st = finalize_device(ctx, s);
  if (st != TSKV_OK) return st;
  if (out_values_dptr) *out_values_dptr = (uint64_t)(uintptr_t)s->d_values.get();
  if (out_validity_dptr) *out_validity_dptr = (uint64_t)(uintptr_t)s->d_validity.get();
  return TSKV_OK;
}

void tskvgpu_scan_destroy(tskv_ctx *ctx, tskv_scan *s) {
  if (ctx) cudaSetDevice(ctx->device);
  delete s;
}

static tskv_status scan_aggregate(tskv_ctx *ctx, const tskv_pages *pages, const tskv_query *q, int64_t slide,
                                  const TagGroups &tg, uint64_t *out_values, uint8_t *out_validity,
                                  const BucketEdges &E = BucketEdges{}) {
  if (!out_values || !out_validity) return TSKV_ERR_INVALID_ARG;
  tskv_scan *s = nullptr;
  tskv_status st = slide ? prepare_sliding(ctx, pages, q, slide, tg, &s) : prepare_scan(ctx, pages, q, 0, tg, &s, E);
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

tskv_status tskvgpu_scan_aggregate_edges(tskv_ctx *ctx, const tskv_pages *pages, const tskv_query *q, const int64_t *edges,
                                         const uint32_t *group_ids, uint32_t n_groups, uint64_t *out_values, uint8_t *out_validity) {
  return scan_aggregate(ctx, pages, q, 0, TagGroups{group_ids != nullptr, group_ids, n_groups}, out_values, out_validity,
                        plain_edges(q, edges));
}

tskv_status tskvgpu_scan_aggregate_labels(tskv_ctx *ctx, const tskv_pages *pages, const tskv_query *q, const int64_t *edges,
                                          uint32_t n_edge, const uint32_t *labels, const uint32_t *group_ids, uint32_t n_groups,
                                          uint64_t *out_values, uint8_t *out_validity) {
  return scan_aggregate(ctx, pages, q, 0, TagGroups{group_ids != nullptr, group_ids, n_groups}, out_values, out_validity,
                        BucketEdges{true, edges, n_edge, true, labels});
}

}  // extern "C"
