// host_util.h — host-side helpers of the C-ABI library: page framing validation, decode-kind
// classification (the codec dispatch of tskv/src/tsm/codec/instance.rs:358-401 done once at upload
// instead of per read), CRC-32/IEEE (tskv/src/tsm/page.rs:58-76).
#pragma once
#include <cstddef>
#include <cstdint>
#include <vector>

#include "../../include/tskv_gpu.h"
#include "kinds.h"

namespace tskv {

// CRC-32/IEEE (crc32fast semantics), slicing-by-8.
uint32_t crc32_ieee(const uint8_t *data, size_t len);
// The slicing-by-8 tables ([8][256]), for the device-side verifier.
const uint32_t *crc32_tables();

struct PageHeader {
  uint32_t bitset_len;
  uint64_t n_rows;
  uint32_t crc;
  const uint8_t *bitset;
  const uint8_t *data;
  uint64_t data_len;
};

// Parses `u32be bitset_len | u64be rows | u32be crc | bitset | data` (page.rs:334-345).
// Returns false when the page is shorter than its own framing.
bool parse_page(const uint8_t *page, uint64_t size, PageHeader *out);

// Decode kind (DK_* of cursors.cuh) of a page of physical type `phys_type`; error kinds encode the
// reference's decode errors so that they surface when (and only when) the page is read.
// ---- scan planning heuristics (host only; exercised on the CPU by tests/test_scan_planning.py) -------------------
// Expected fraction of an arena's series a query selects. The id list may cover more than this arena (a multi-GPU
// caller hands the whole selection to every shard): only ids inside the arena's id range can match.
// Both lists sorted ascending; n_sel == 0 with sel == nullptr means "all series".
double plan_selected_fraction(const uint32_t *arena_series, uint64_t n_arena, const uint32_t *sel, uint64_t n_sel);
// Grid sizes of the lane-per-page kernels of one scan (one persistent kernel per decode-kind bin, all launched
// concurrently; a warp repeatedly takes a chunk of 32 pages of its bin). A chunk is ONE serial task of t_chunk[b]
// (relative units: rows x cost of the bin's codec pair), so a bin finishes after ceil(chunks / warps) rounds of
// t_chunk: the makespan is quantised. Picks the smallest makespan T for which giving every bin
// ceil(chunks_b / (floor(T / t_b) * warps_per_block)) blocks fits the machine, sum_b blocks_b / occ_b <= sm_count
// (a block of bin b takes 1/occ_b of an SM). Bins with chunks[b] == 0 get 0 blocks.
void plan_serial_grids(int n_bins, const double *chunks, const double *t_chunk, const int *occ, int sm_count,
                       int warps_per_block, int *grid_out);

// Pages cut at restart points: how many parts per page a scan wants so that it has about `target` chunks (32 pages x
// 1 part) per resident warp - est_chunks = the scan's chunks with whole pages.
uint32_t plan_parts_wanted(double est_chunks, double resident_warps, double target);
// Parts of a bin whose longest page has `maxrows` rows when `want` parts are wanted: parts are whole multiples of the
// restart interval (`skip_rows` rows), at most one part per interval. Returns the parts; *part_rows = rows per part.
uint32_t plan_bin_parts(uint32_t maxrows, uint32_t skip_rows, uint32_t want, uint32_t *part_rows);
// Threads S per walked series of the work-list walk (a power of two): the smallest S that leaves each thread at most 32
// of the `max_groups` column groups of the page set's largest series, at most 1024, then halved while the walk would
// launch more threads than max(n_items, min_threads) (n_walk = the series walked: selected ids or every series).
uint32_t plan_walk_split(uint32_t max_groups, uint64_t n_walk, uint64_t n_items, uint32_t min_threads);
// Does a page set whose n_series distinct ids span [min_id, max_id] get a direct id -> rank table (4 bytes per id of
// the span) instead of a binary search? Yes when the span is at most 2 x n_series + SERIES_MAP_SLACK ids: the table then
// costs at most twice the sorted id list plus 64 KB.
constexpr uint64_t SERIES_MAP_SLACK = 16384;
bool plan_series_map(uint32_t min_id, uint32_t max_id, uint64_t n_series);
// Work-list regions: bucket k gets [start[k], start[k] + capacity[k]), every start a multiple of 32 (one chunk of the
// fused kernels never holds items of two buckets). start has n_buckets + 1 entries; start[n_buckets] = the list's size.
// Returns false when the list would not fit 32-bit item indices.
bool plan_worklist_regions(uint32_t n_buckets, const uint32_t *capacity, uint32_t *start);

uint8_t classify_page(const PageHeader &h, uint8_t phys_type);

// ---- overlapping chunks (reader/iterator.rs:463-560, reader/utils.rs:77-107) --------------------------------------
// A chunk = the column groups of one series that come from one file. Per series: chunks sorted by time range, grouped
// while a chunk starts at or before the running maximum end (group_overlapping_segments), each group ordered by file
// id. Groups of more than one chunk are MERGE GROUPS: their column groups leave the normal work list and go through
// the merge pass (merge_kernels.cuh). The plan lays the merge groups' rows out stream by stream (stream = one chunk,
// its column groups in time order), so every stream is one time-sorted run of consecutive merge rows.
struct OverlapPlan {
  std::vector<uint8_t> cg_merge;          // [n_cg] 1: the column group belongs to a merge group
  std::vector<uint32_t> mcg_cg;           // merge column groups in merge-row order -> column group index
  std::vector<uint32_t> mcg_stream;       // -> stream index
  std::vector<uint64_t> mcg_row0;         // [n_mcg + 1] first merge row of each merge column group
  std::vector<uint32_t> stream_group;     // [n_streams] -> merge group
  std::vector<uint32_t> stream_first_mcg; // [n_streams + 1]
  std::vector<uint32_t> group_first_stream;  // [n_groups + 1]
  uint64_t n_groups_total = 0;            // overlap groups of all series, merge groups or not (the reference's metric)
};
void plan_overlap_groups(uint64_t n_cg, const uint32_t *cg_series, const uint32_t *cg_rows, const tskv_time_range *cg_bounds,
                         const uint64_t *cg_file, OverlapPlan *out);

}  // namespace tskv
