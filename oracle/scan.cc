// oracle/scan.cc — CPU restatement of the reference scan: per series, per column group decode
// (tsm/reader.rs:494-560) -> closed time-range filter (predicate/domain.rs:35-98, reader/filter.rs)
// -> bucket key (transform_time_window.rs:251-296) -> aggregates (DataFusion builtins + first.rs /
// last.rs semantics). TEST INFRASTRUCTURE ONLY (see tskv_oracle.h).
#include <algorithm>
#include <condition_variable>
#include <cstring>
#include <functional>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "tskv_oracle.h"

namespace {

thread_local std::string g_err;
bool g_value_stats_pruning = true;  // orc_set_value_stats_pruning (tests compare pruned and unpruned scans)


// `sliding_window` (query_server/query/src/extension/expr/window/time_window.rs:184-198); Rust `%`
// keeps the sign of the dividend, like C; release builds wrap on overflow.
inline void sliding_window(int64_t t, int64_t w, int64_t s, int64_t start_time, int64_t i,
                           int64_t *ws, int64_t *we) {
  int64_t st = start_time % w;
  int64_t dividend = (int64_t)((uint64_t)t - (uint64_t)st + (uint64_t)s);
  int64_t last_start = (int64_t)((uint64_t)t - (uint64_t)(dividend % s));
  *ws = (int64_t)((uint64_t)last_start - (uint64_t)i * (uint64_t)s);
  *we = (int64_t)((uint64_t)*ws + (uint64_t)w);
}

// Total order on f64 bit patterns (NaN handling of DataFusion min/max is unpinned in the
// reference tree; the f64 edge tests aggregate NaNs of both signs and check MIN / MAX under this order).
inline int64_t f64_okey(uint64_t b) { return (int64_t)(b ^ (((int64_t)b >> 63) & 0x7fffffffffffffffll)); }

inline bool less_typed(uint8_t pt, uint64_t a, uint64_t b) {
  if (pt == TSKV_PT_I64) return (int64_t)a < (int64_t)b;
  if (pt == TSKV_PT_U64 || pt == TSKV_PT_BOOL) return a < b;
  return f64_okey(a) < f64_okey(b);
}

// One `column <op> constant` of the pushed row filter (reader/filter.rs:130-142: the predicate is evaluated on the
// schema-aligned batch and applied with filter_record_batch, which keeps a row only where the predicate is TRUE).
inline bool cmp_true(uint8_t pt, uint8_t op, uint64_t v, uint64_t c) {
  int r;  // -1 / 0 / +1, or 2 for unordered (NaN)
  if (pt == TSKV_PT_I64) r = (int64_t)v < (int64_t)c ? -1 : ((int64_t)v > (int64_t)c ? 1 : 0);
  else if (pt == TSKV_PT_U64) r = v < c ? -1 : (v > c ? 1 : 0);
  else {
    double a, b;
    memcpy(&a, &v, 8);
    memcpy(&b, &c, 8);
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

struct Cell {
  uint64_t count = 0;
  uint64_t sum_bits = 0;  // i64/u64 wrapping sum
  double sum_d = 0.0;     // f64 sum (arrival order); for ints: sum of values cast to f64 (avg)
  uint64_t minv = 0, maxv = 0;
  bool has_first = false, has_last = false;
  int64_t first_ts = 0, last_ts = 0;
  uint64_t first_val = 0, last_val = 0;
};

struct ColumnGroup {
  uint64_t first_desc;  // the TIME page
  uint64_t n_descs;     // incl. the time page
  uint64_t orig;        // index of the column group in descriptor-table order
  int64_t min_ts;       // first time value (orders the column groups of a chunk; filled by orc_set_chunk_files)
};

struct SeriesGroups {
  uint32_t series;
  uint32_t first_cg, n_cg;  // range in Index::cgs
};
struct Index {
  std::vector<uint32_t> series;       // sorted distinct ids
  std::vector<ColumnGroup> cgs;       // column groups, sorted by (series, arena order)
  std::vector<SeriesGroups> by_series;  // sorted by series id
  // column groups of one series (arena order), or an empty range
  std::pair<const ColumnGroup *, const ColumnGroup *> find(uint32_t sid) const {
    size_t lo = 0, hi = by_series.size();
    while (lo < hi) {
      size_t mid = (lo + hi) / 2;
      if (by_series[mid].series < sid) lo = mid + 1; else hi = mid;
    }
    if (lo == by_series.size() || by_series[lo].series != sid) return {nullptr, nullptr};
    const ColumnGroup *b = cgs.data() + by_series[lo].first_cg;
    return {b, b + by_series[lo].n_cg};
  }
};

tskv_status build_index(const tskv_page_desc *descs, uint64_t n, Index &ix) {
  uint64_t i = 0;
  while (i < n) {
    if (descs[i].phys_type != TSKV_PT_TIME) {
      g_err = "descriptor table: column group does not start with a time page";
      return TSKV_ERR_INVALID_ARG;
    }
    uint64_t j = i + 1;
    while (j < n && descs[j].phys_type != TSKV_PT_TIME) {
      if (descs[j].series_id != descs[i].series_id || descs[j].num_values != descs[i].num_values) {
        g_err = "descriptor table: field page disagrees with its time page";
        return TSKV_ERR_INVALID_ARG;
      }
      j++;
    }
    ix.cgs.push_back(ColumnGroup{i, j - i, (uint64_t)ix.cgs.size(), 0});
    i = j;
  }
  // group by series keeping the arena order inside a series (compacted files are already sorted)
  auto sid = [&](const ColumnGroup &c) { return descs[c.first_desc].series_id; };
  bool sorted = true;
  for (size_t k = 1; k < ix.cgs.size() && sorted; k++) sorted = sid(ix.cgs[k - 1]) <= sid(ix.cgs[k]);
  if (!sorted) std::stable_sort(ix.cgs.begin(), ix.cgs.end(), [&](const ColumnGroup &a, const ColumnGroup &b) { return sid(a) < sid(b); });
  for (size_t k = 0; k < ix.cgs.size(); k++) {
    uint32_t s = sid(ix.cgs[k]);
    if (ix.by_series.empty() || ix.by_series.back().series != s) {
      ix.by_series.push_back(SeriesGroups{s, (uint32_t)k, 0});
      ix.series.push_back(s);
    }
    ix.by_series.back().n_cg++;
  }
  return TSKV_OK;
}

inline unsigned popc(unsigned x) { return (unsigned)__builtin_popcount(x); }

struct Scan {
  const uint8_t *arena;
  uint64_t arena_len;
  const tskv_page_desc *descs;
  const tskv_query *q;
  int verify_crc;
  const Index *ix;
  std::vector<uint32_t> slots;  // slot -> series id
  uint64_t n_cells;
  const tskv_tombstone *tombs = nullptr;
  uint64_t n_tombs = 0;
  const uint64_t *cg_file = nullptr;  // file id of every column group (descriptor-table order), or null: one file
  bool value_stats_pruning = true;
};

// update_nullbits_by_time_range (tsm/reader.rs:634-656): binary search over the page's time VALUES (the raw
// value buffer, nulls included) for [min_ts, max_ts]; clears bits start..end.
void clear_bits_by_time_range(const std::vector<uint64_t> &ts, uint64_t n_rows, int64_t min_ts, int64_t max_ts,
                              std::vector<uint8_t> &bits) {
  auto lower = [&](int64_t x, bool *found) {  // slice::binary_search: Ok(i) if found else Err(insertion point)
    uint64_t lo = 0, hi = n_rows;
    *found = false;
    while (lo < hi) {
      uint64_t mid = lo + (hi - lo) / 2;
      int64_t v = (int64_t)ts[mid];
      if (v == x) { *found = true; return mid; }
      if (v < x) lo = mid + 1;
      else hi = mid;
    }
    return lo;
  };
  bool f;
  uint64_t start = lower(min_ts, &f);
  uint64_t end = lower(max_ts, &f);
  if (f) end += 1;
  for (uint64_t i = start; i < end && i < n_rows; i++) bits[i] = 0;
}

// ---- overlapping chunks (reader/iterator.rs:463-560, reader/utils.rs:77-107, reader/sort_merge.rs, reader/batch_builder.rs)
// A chunk = the column groups of one series in one file (tsm/chunk.rs); the caller tags every column group with the id
// of the file it came from (orc_set_chunk_files). Per series the reference sorts the chunks by time range, groups the
// ones whose ranges overlap (group_overlapping_segments), orders each group by file id and - for a group of more than
// one chunk - k-way merges the chunks' row streams on `time` (DataMerger -> sort_merge): ties go to the lower stream
// index, rows with equal time collapse into one whose every column takes the LAST non-null value in arrival order
// (BatchMergeBuilder::take_last_and_merge), the first row's null otherwise.
struct ChunkRef {
  uint64_t file_id;
  int64_t min_ts, max_ts;
  std::vector<const ColumnGroup *> cgs;
};

struct Worker {
  const Scan &S;
  Cell *cells;
  uint64_t *points;
  std::vector<uint64_t> ts, vals, pvals;
  std::vector<uint8_t> tvalid, vvalid, keep, pred_keep, pvalid;
  bool have_keep = false;
  int64_t page_min = 0, page_max = 0;
  Worker(const Scan &s, Cell *c, uint64_t *p) : S(s), cells(c), points(p) {}

  // Decodes the time page of a column group and evaluates what filters its ROWS: statistics pruning, the pushed
  // predicates, the all-fields tombstones. `pruned` = the group is never read.
  tskv_status prepare_cg(const ColumnGroup &cg, bool *pruned) {
    const tskv_query &q = *S.q;
    const tskv_page_desc &td = S.descs[cg.first_desc];
    const uint64_t n_rows = td.num_values;
    *pruned = false;
    ts.assign(n_rows ? n_rows : 1, 0);
    tvalid.assign(n_rows ? n_rows : 1, 0);
    uint64_t nr = 0;
    if (td.offset + td.size > S.arena_len) return TSKV_ERR_INVALID_ARG;
    tskv_status st = orc_page_decode(TSKV_PT_TIME, S.arena + td.offset, td.size, S.verify_crc,
                                     ts.data(), tvalid.data(), n_rows, &nr);
    if (st != TSKV_OK) return st;
    if (nr != n_rows) return TSKV_ERR_PAGE_FORMAT;
    // Statistics pruning (filter_column_groups, tskv/src/reader/chunk.rs:12-50): a column group whose time range
    // (ColumnGroup::time_range(), here: min / max of its time values) overlaps none of the query's ranges is never
    // read - its field pages are neither decoded nor counted.
    if (q.n_time_ranges && n_rows) {
      int64_t gmin = INT64_MAX, gmax = INT64_MIN;
      for (uint64_t r = 0; r < n_rows; r++)
        if (tvalid[r]) { gmin = std::min(gmin, (int64_t)ts[r]); gmax = std::max(gmax, (int64_t)ts[r]); }
      bool overlaps = false;
      for (uint32_t k = 0; k < q.n_time_ranges; k++)
        overlaps = overlaps || (gmin <= q.time_ranges[k].max_ts && gmax >= q.time_ranges[k].min_ts);
      if (!overlaps) { *pruned = true; return TSKV_OK; }
    }
    // the row filter: every predicate column of this column group decoded, rows kept where all comparisons are TRUE;
    // a column the group does not hold is null-filled by SchemaAlignmenter (schema_alignmenter.rs:24-44) => no row passes
    pred_keep.assign(n_rows ? n_rows : 1, 1);
    for (uint32_t k = 0; k < q.n_predicates; k++) {
      const tskv_field_predicate &fp = q.predicates[k];
      const tskv_page_desc *pd = nullptr;
      for (uint64_t j = 1; j < cg.n_descs; j++)
        if (S.descs[cg.first_desc + j].column_id == fp.column_id) {
          pd = &S.descs[cg.first_desc + j];
          break;
        }
      if (!pd) {
        std::fill(pred_keep.begin(), pred_keep.end(), (uint8_t)0);
        continue;
      }
      if (pd->phys_type != fp.phys_type) {
        g_err = "page type does not match the predicate column type";
        return TSKV_ERR_INVALID_ARG;
      }
      pvals.assign(n_rows ? n_rows : 1, 0);
      pvalid.assign(n_rows ? n_rows : 1, 0);
      uint64_t pr = 0;
      tskv_status pst = orc_page_decode(pd->phys_type, S.arena + pd->offset, pd->size, S.verify_crc, pvals.data(),
                                        pvalid.data(), n_rows, &pr);
      if (pst != TSKV_OK) return pst;
      // Value statistics (filter_column_groups -> PruningPredicate over PageMeta.statistics, reader/chunk.rs:12-50,
      // reader/column_group/statistics.rs:11-80): when the page's min / max rule the comparison out for every row, the
      // column group is never read. min / max over the non-null, non-NaN values; -0.0 counts as +0.0.
      {
        bool have = false;
        uint64_t vmin = 0, vmax = 0;
        for (uint64_t r = 0; r < n_rows; r++) {
          if (!pvalid[r]) continue;
          uint64_t v = pvals[r];
          if (fp.phys_type == TSKV_PT_F64) {
            if ((v & 0x7fffffffffffffffull) > 0x7ff0000000000000ull) continue;
            if (v == 0x8000000000000000ull) v = 0;
          }
          if (!have) { vmin = vmax = v; have = true; }
          else {
            if (less_typed(fp.phys_type, v, vmin)) vmin = v;
            if (less_typed(fp.phys_type, vmax, v)) vmax = v;
          }
        }
        uint64_t c = fp.value;
        bool nan_const = fp.phys_type == TSKV_PT_F64 && (c & 0x7fffffffffffffffull) > 0x7ff0000000000000ull;
        if (fp.phys_type == TSKV_PT_F64 && c == 0x8000000000000000ull) c = 0;
        bool out = !have || nan_const;
        if (!out) {
          const bool c_lt_min = less_typed(fp.phys_type, c, vmin), c_gt_max = less_typed(fp.phys_type, vmax, c);
          switch (fp.op) {
            case TSKV_CMP_EQ: out = c_lt_min || c_gt_max; break;
            case TSKV_CMP_NE: out = vmin == vmax && vmin == c; break;
            case TSKV_CMP_LT: out = !less_typed(fp.phys_type, vmin, c); break;   // min >= c
            case TSKV_CMP_LE: out = c_lt_min; break;                              // min > c
            case TSKV_CMP_GT: out = !less_typed(fp.phys_type, c, vmax); break;   // max <= c
            case TSKV_CMP_GE: out = c_gt_max; break;                              // max < c
            default: break;
          }
        }
        if (out && S.value_stats_pruning) { *pruned = true; return TSKV_OK; }
      }
      for (uint64_t r = 0; r < n_rows; r++)
        if (!(pvalid[r] && cmp_true(fp.phys_type, fp.op, pvals[r], fp.value))) pred_keep[r] = 0;
    }
    // decode_pages with a tombstone (reader.rs:507-524): the all-fields excluded ranges that overlap the
    // page's time range clear bits of the TIME page's null bitset; the result filters the rows.
    keep.assign(n_rows ? n_rows : 1, 1);
    have_keep = false;
    if (S.n_tombs && n_rows) {
      int64_t pmin = INT64_MAX, pmax = INT64_MIN;  // PageStatistics min/max of the time column
      for (uint64_t r = 0; r < n_rows; r++)
        if (tvalid[r]) { pmin = std::min(pmin, (int64_t)ts[r]); pmax = std::max(pmax, (int64_t)ts[r]); }
      page_min = pmin; page_max = pmax;
      for (uint64_t k = 0; k < S.n_tombs; k++) {
        const tskv_tombstone &tb = S.tombs[k];
        if (tb.column_id != TSKV_TOMB_ALL) continue;
        if (tb.series_id != TSKV_TOMB_ALL && tb.series_id != td.series_id) continue;
        if (!(tb.min_ts <= pmax && tb.max_ts >= pmin)) continue;  // TimeRange::overlaps
        if (!have_keep) { keep = tvalid; have_keep = true; }
        clear_bits_by_time_range(ts, n_rows, tb.min_ts, tb.max_ts, keep);
      }
    }
    return TSKV_OK;
  }

  // Decodes one field page of the prepared column group into vals / vvalid (per-column tombstones applied).
  tskv_status load_field(const tskv_page_desc *fd, uint64_t n_rows) {
    vals.assign(n_rows ? n_rows : 1, 0);
    vvalid.assign(n_rows ? n_rows : 1, 0);
    uint64_t nr = 0;
    if (fd->offset + fd->size > S.arena_len) return TSKV_ERR_INVALID_ARG;
    tskv_status st = orc_page_decode(fd->phys_type, S.arena + fd->offset, fd->size, S.verify_crc,
                                     vals.data(), vvalid.data(), n_rows, &nr);
    if (st != TSKV_OK) return st;
    if (nr != n_rows) return TSKV_ERR_PAGE_FORMAT;
    // per-column tombstones (reader.rs:531-542): clear the value validity of the excluded rows
    for (uint64_t k = 0; k < S.n_tombs && n_rows; k++) {
      const tskv_tombstone &tb = S.tombs[k];
      if (tb.column_id == TSKV_TOMB_ALL || tb.series_id != fd->series_id || tb.column_id != fd->column_id) continue;
      if (!(tb.min_ts <= page_max && tb.max_ts >= page_min)) continue;
      clear_bits_by_time_range(ts, n_rows, tb.min_ts, tb.max_ts, vvalid);
    }
    return TSKV_OK;
  }

  const tskv_page_desc *find_field(const ColumnGroup &cg, const tskv_agg_column &qc, tskv_status *st) {
    *st = TSKV_OK;
    for (uint64_t k = 1; k < cg.n_descs; k++)
      if (S.descs[cg.first_desc + k].column_id == qc.column_id) {
        const tskv_page_desc *fd = &S.descs[cg.first_desc + k];
        if (fd->phys_type != qc.phys_type) {
          g_err = "page type does not match the query column type";
          *st = TSKV_ERR_INVALID_ARG;
        }
        return fd;
      }
    return nullptr;  // column absent from this column group (null-filled by SchemaAlignmenter)
  }

  // The rows of one record batch into the cells of query column c: row keep flags (null: all kept), closed time
  // ranges, bucket key, aggregates.
  tskv_status aggregate_rows(uint32_t c, uint64_t group, uint64_t n_rows, const uint64_t *bts, const uint8_t *btvalid,
                             const uint64_t *bvals, const uint8_t *bvvalid, const uint8_t *row_keep,
                             const uint8_t *row_pred) {
    const tskv_query &q = *S.q;
    const tskv_agg_column &qc = q.columns[c];
    const uint8_t pt = qc.phys_type;
    Cell *ccells = cells + (uint64_t)c * S.n_cells + group * q.n_buckets;
    // Run state for first/last: the rows of one (page, bucket) form one DataFusion group slice;
    // FirstAccumulator::update_batch picks its min-time row and drops it when the VALUE is null
    // (first.rs:139-148 + :91-94). Pages are time-sorted (mem_cache/series_data.rs:218-262), so a
    // (page, bucket) group is one contiguous run of rows.
    int64_t run_bucket = -1;
    uint64_t run_first = 0, run_last = 0;
    auto close_run = [&]() {
      if (run_bucket < 0) return;
      Cell &cell = ccells[run_bucket];
      if ((qc.agg_mask & TSKV_AGG_FIRST) && bvvalid[run_first]) {
        int64_t t = (int64_t)bts[run_first];
        if (!cell.has_first || t < cell.first_ts) {  // strictly less: ties keep the earlier-seen
          cell.has_first = true;
          cell.first_ts = t;
          cell.first_val = bvals[run_first];
        }
      }
      if ((qc.agg_mask & TSKV_AGG_LAST) && bvvalid[run_last]) {
        int64_t t = (int64_t)bts[run_last];
        if (!cell.has_last || t > cell.last_ts) {
          cell.has_last = true;
          cell.last_ts = t;
          cell.last_val = bvals[run_last];
        }
      }
    };
    for (uint64_t r = 0; r < n_rows; r++) {
      if (row_keep && !row_keep[r]) continue;  // filter_record_batch(&record_batch, time_null_bits) (reader.rs:546-550)
      if (row_pred && !row_pred[r]) continue;  // DataFilter (reader/filter.rs:130-142)
      if (!btvalid[r]) continue;  // is_not_null(time) (transform_time_window.rs:313)
      int64_t t = (int64_t)bts[r];
      bool in = q.n_time_ranges == 0;
      for (uint32_t k = 0; k < q.n_time_ranges && !in; k++)
        in = t >= q.time_ranges[k].min_ts && t <= q.time_ranges[k].max_ts;  // TimeRange::contains
      if (!in) continue;
      int64_t b = 0;
      if (q.width > 0) {
        int64_t ws, we;
        sliding_window(t, q.width, q.width, q.origin, 0, &ws, &we);
        int64_t diff = (int64_t)((uint64_t)ws - (uint64_t)q.first_bucket_start);
        if (diff < 0 || diff % q.width != 0 || diff / q.width >= (int64_t)q.n_buckets) {
          g_err = "row outside the requested bucket range";
          return TSKV_ERR_BUCKET_RANGE;
        }
        b = diff / q.width;
      }
      if (b != run_bucket) {
        close_run();
        run_bucket = b;
        run_first = run_last = r;
      } else {
        if ((int64_t)bts[r] < (int64_t)bts[run_first]) run_first = r;
        if ((int64_t)bts[r] > (int64_t)bts[run_last]) run_last = r;
      }
      if (!bvvalid[r]) continue;
      Cell &cell = ccells[b];
      uint64_t v = bvals[r];
      if (cell.count == 0) {
        cell.minv = cell.maxv = v;
      } else {
        if (less_typed(pt, v, cell.minv)) cell.minv = v;
        if (less_typed(pt, cell.maxv, v)) cell.maxv = v;
      }
      cell.count++;
      if (pt == TSKV_PT_F64) {
        double d;
        memcpy(&d, &v, 8);
        cell.sum_d += d;
      } else {
        cell.sum_bits += v;
        cell.sum_d += pt == TSKV_PT_I64 ? (double)(int64_t)v : (double)v;
      }
    }
    close_run();
    return TSKV_OK;
  }

  // One column group read on its own (no overlapping chunk): ColumnGroupReader -> DataFilter -> aggregate.
  tskv_status scan_cg(const ColumnGroup &cg, uint64_t group) {
    const tskv_query &q = *S.q;
    const uint64_t n_rows = S.descs[cg.first_desc].num_values;
    bool prepared = false, pruned = false;
    for (uint32_t c = 0; c < q.n_columns && !pruned; c++) {
      tskv_status st;
      const tskv_page_desc *fd = find_field(cg, q.columns[c], &st);
      if (st != TSKV_OK) return st;
      if (!fd) continue;
      if (!prepared) {
        st = prepare_cg(cg, &pruned);
        if (st != TSKV_OK) return st;
        prepared = true;
        if (pruned) break;
      }
      st = load_field(fd, n_rows);
      if (st != TSKV_OK) return st;
      if (points)
        for (uint64_t r = 0; r < n_rows; r++)
          if (vvalid[r]) (*points)++;
      st = aggregate_rows(c, group, n_rows, ts.data(), tvalid.data(), vals.data(), vvalid.data(),
                          have_keep ? keep.data() : nullptr, q.n_predicates ? pred_keep.data() : nullptr);
      if (st != TSKV_OK) return st;
    }
    return TSKV_OK;
  }

  // A group of overlapping chunks, ordered by file id: every chunk is one sorted row stream (its column groups in time
  // order, each filtered like scan_cg would), schema-aligned to time + the query's columns; the streams are merged
  // and de-duplicated as described above, and the merged rows form ONE record batch (the reference cuts batches of
  // `batch_size` rows; the cut only matters to first / last when the first / last row of a batch holds a NULL).
  tskv_status scan_merged(const std::vector<const ChunkRef *> &streams, uint64_t group) {
    const tskv_query &q = *S.q;
    struct Row { int64_t t; uint32_t stream; };
    const uint32_t nc = q.n_columns;
    std::vector<int64_t> rt;                 // row time
    std::vector<uint32_t> rs;                // row stream
    std::vector<std::vector<uint64_t>> rv(nc);
    std::vector<std::vector<uint8_t>> rok(nc);
    for (uint32_t si = 0; si < streams.size(); si++) {
      for (const ColumnGroup *cgp : streams[si]->cgs) {
        const ColumnGroup &cg = *cgp;
        const uint64_t n_rows = S.descs[cg.first_desc].num_values;
        bool any = false;
        std::vector<const tskv_page_desc *> fds(nc, nullptr);
        for (uint32_t c = 0; c < nc; c++) {
          tskv_status st;
          fds[c] = find_field(cg, q.columns[c], &st);
          if (st != TSKV_OK) return st;
          any = any || fds[c];
        }
        if (!any) continue;  // (a column group without any projected column yields no batch: column_group/mod.rs:43-52)
        bool pruned = false;
        tskv_status st = prepare_cg(cg, &pruned);
        if (st != TSKV_OK) return st;
        if (pruned) continue;
        const size_t base = rt.size();
        std::vector<uint64_t> sel;  // rows of this column group that reach the merge
        for (uint64_t r = 0; r < n_rows; r++) {
          if (have_keep && !keep[r]) continue;
          if (q.n_predicates && !pred_keep[r]) continue;
          if (!tvalid[r]) continue;
          sel.push_back(r);
          rt.push_back((int64_t)ts[r]);
          rs.push_back(si);
        }
        for (uint32_t c = 0; c < nc; c++) {
          rv[c].resize(base + sel.size(), 0);
          rok[c].resize(base + sel.size(), 0);
          if (!fds[c]) continue;
          st = load_field(fds[c], n_rows);
          if (st != TSKV_OK) return st;
          if (points)
            for (uint64_t r = 0; r < n_rows; r++)
              if (vvalid[r]) (*points)++;
          for (size_t k = 0; k < sel.size(); k++) {
            rv[c][base + k] = vvalid[sel[k]] ? vals[sel[k]] : 0;
            rok[c][base + k] = vvalid[sel[k]];
          }
        }
      }
    }
    // k-way merge on time, ties to the lower stream index then the earlier row (sort_merge.rs:300-306): the rows were
    // appended stream by stream in row order, so a STABLE sort by time is that order
    std::vector<uint32_t> order(rt.size());
    for (uint32_t i = 0; i < order.size(); i++) order[i] = i;
    for (size_t i = 1; i < rt.size(); i++)
      if (rs[i] == rs[i - 1] && rt[i] < rt[i - 1]) {
        g_err = "data in stream is not sorted";  // batch_builder.rs:121-126
        return TSKV_ERR_INVALID_ARG;
      }
    std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return rt[a] < rt[b]; });
    std::vector<uint64_t> mts;
    std::vector<uint8_t> mtvalid;
    std::vector<std::vector<uint64_t>> mv(nc);
    std::vector<std::vector<uint8_t>> mok(nc);
    for (size_t i = 0; i < order.size();) {
      size_t j = i;
      while (j < order.size() && rt[order[j]] == rt[order[i]]) j++;
      mts.push_back((uint64_t)rt[order[i]]);
      mtvalid.push_back(1);
      for (uint32_t c = 0; c < nc; c++) {  // take_last_and_merge (batch_builder.rs:133-155)
        uint64_t v = 0;
        uint8_t ok = 0;
        for (size_t k = j; k-- > i;)
          if (rok[c][order[k]]) { v = rv[c][order[k]]; ok = 1; break; }
        mv[c].push_back(v);
        mok[c].push_back(ok);
      }
      i = j;
    }
    for (uint32_t c = 0; c < nc; c++) {
      tskv_status st = aggregate_rows(c, group, mts.size(), mts.data(), mtvalid.data(), mv[c].data(), mok[c].data(), nullptr, nullptr);
      if (st != TSKV_OK) return st;
    }
    return TSKV_OK;
  }
};

// group_overlapping_segments (reader/utils.rs:77-107) over chunks sorted by time range.
std::vector<std::vector<const ChunkRef *>> group_overlapping(const std::vector<ChunkRef> &sorted) {
  std::vector<std::vector<const ChunkRef *>> out;
  int64_t global_max = INT64_MIN;  // (named global_min_ts in the reference)
  for (const ChunkRef &ch : sorted) {
    if (!out.empty() && ch.min_ts <= global_max) out.back().push_back(&ch);
    else out.push_back({&ch});
    global_max = std::max(ch.max_ts, global_max);
  }
  return out;
}

// One worker: slots [s0, s1) into `cells` (n_columns * n_cells). Returns status.
tskv_status scan_slots(const Scan &S, uint64_t s0, uint64_t s1, Cell *cells, bool shared_table,
                       uint64_t *points) {
  const tskv_query &q = *S.q;
  (void)shared_table;
  Worker W(S, cells, points);
  for (uint64_t slot = s0; slot < s1; slot++) {
    auto range = S.ix->find(S.slots[slot]);
    if (range.first == nullptr) continue;  // selected id absent from this arena
    const uint64_t group = q.group_by_series ? slot : 0;
    if (!S.cg_file) {  // one file: its column groups in arena order
      for (const ColumnGroup *cgp = range.first; cgp != range.second; cgp++) {
        tskv_status st = W.scan_cg(*cgp, group);
        if (st != TSKV_OK) return st;
      }
      continue;
    }
    // several files (build_series_reader, reader/iterator.rs:463-560): chunks = column groups by file id
    std::vector<ChunkRef> chunks;
    for (const ColumnGroup *cgp = range.first; cgp != range.second; cgp++) {
      const uint64_t fid = S.cg_file[cgp->orig];
      ChunkRef *ch = nullptr;
      for (ChunkRef &c : chunks)
        if (c.file_id == fid) ch = &c;
      if (!ch) {
        chunks.push_back(ChunkRef{fid, INT64_MAX, INT64_MIN, {}});
        ch = &chunks.back();
      }
      // ColumnGroup::time_range(): min / max of the time values
      const tskv_page_desc &td = S.descs[cgp->first_desc];
      std::vector<uint64_t> t(td.num_values ? td.num_values : 1);
      std::vector<uint8_t> tv(td.num_values ? td.num_values : 1);
      uint64_t nr = 0;
      tskv_status st = orc_page_decode(TSKV_PT_TIME, S.arena + td.offset, td.size, 0, t.data(), tv.data(), td.num_values, &nr);
      if (st != TSKV_OK) return st;
      for (uint64_t r = 0; r < nr; r++)
        if (tv[r]) { ch->min_ts = std::min(ch->min_ts, (int64_t)t[r]); ch->max_ts = std::max(ch->max_ts, (int64_t)t[r]); }
      ch->cgs.push_back(cgp);
    }
    for (ChunkRef &ch : chunks)  // a chunk's column groups in time order (Chunk::push keeps them so, tsm/chunk.rs:100-110)
      std::stable_sort(ch.cgs.begin(), ch.cgs.end(), [&](const ColumnGroup *a, const ColumnGroup *b) { return a->min_ts < b->min_ts; });
    // chunks.sort_unstable_by_key(|e| e.time_range()): (min_ts, max_ts); equal ranges: by file id, for determinism
    std::sort(chunks.begin(), chunks.end(), [](const ChunkRef &a, const ChunkRef &b) {
      if (a.min_ts != b.min_ts) return a.min_ts < b.min_ts;
      if (a.max_ts != b.max_ts) return a.max_ts < b.max_ts;
      return a.file_id < b.file_id;
    });
    auto groups = group_overlapping(chunks);
    for (auto &g : groups) {
      std::stable_sort(g.begin(), g.end(), [](const ChunkRef *a, const ChunkRef *b) { return a->file_id < b->file_id; });  // g.sort()
      tskv_status st = TSKV_OK;
      if (g.size() == 1) {
        for (const ColumnGroup *cgp : g[0]->cgs) {
          st = W.scan_cg(*cgp, group);
          if (st != TSKV_OK) return st;
        }
      } else {
        st = W.scan_merged(g, group);
        if (st != TSKV_OK) return st;
      }
    }
  }
  return TSKV_OK;
}

void merge_cell(Cell &a, const Cell &b, uint8_t pt) {
  if (b.count) {
    if (a.count == 0) {
      a.minv = b.minv;
      a.maxv = b.maxv;
    } else {
      if (less_typed(pt, b.minv, a.minv)) a.minv = b.minv;
      if (less_typed(pt, a.maxv, b.maxv)) a.maxv = b.maxv;
    }
    a.count += b.count;
    a.sum_bits += b.sum_bits;
    a.sum_d += b.sum_d;
  }
  if (b.has_first && (!a.has_first || b.first_ts < a.first_ts)) {
    a.has_first = true;
    a.first_ts = b.first_ts;
    a.first_val = b.first_val;
  }
  if (b.has_last && (!a.has_last || b.last_ts > a.last_ts)) {
    a.has_last = true;
    a.last_ts = b.last_ts;
    a.last_val = b.last_val;
  }
}

}  // namespace

extern "C" {

const char *orc_last_error(void) { return g_err.c_str(); }
void orc_set_value_stats_pruning(int on) { g_value_stats_pruning = on != 0; }

void orc_sliding_window(int64_t t, int64_t window, int64_t slide, int64_t start_time, int64_t i,
                        int64_t *out_start, int64_t *out_end) {
  sliding_window(t, window, slide, start_time, i, out_start, out_end);
}

// time_window.rs:97-147
void orc_ceil_sliding_window(int64_t t, int64_t window, int64_t slide, int64_t start_time,
                             int64_t *out_start, int64_t *out_end) {
  int64_t overlapping = (window + slide - 1) / slide;
  int64_t cs = 0, ce = 0;
  bool have = false;
  for (int64_t i = overlapping - 1; i >= 0; i--) {
    int64_t s, e;
    sliding_window(t, window, slide, start_time, i, &s, &e);
    if (t >= s && t < e) {
      *out_start = s;
      *out_end = e;
      return;
    }
    cs = s;
    ce = e;
    have = true;
  }
  if (have) {
    while (t >= ce) {
      cs += slide;
      ce += slide;
    }
  }
  *out_start = cs;
  *out_end = ce;
}

// time_window.rs:151-182
void orc_floor_sliding_window(int64_t t, int64_t window, int64_t slide, int64_t start_time,
                              int64_t *out_start, int64_t *out_end) {
  int64_t s, e;
  sliding_window(t, window, slide, start_time, 0, &s, &e);
  if (!(t >= s && t < e)) {
    while (t < s) {
      s -= slide;
      e -= slide;
    }
  }
  *out_start = s;
  *out_end = e;
}

tskv_status orc_query_output_layout(const tskv_page_desc *descs, uint64_t n_descs,
                                    const tskv_query *q, tskv_output_layout *out) {
  if (!q || !out || q->n_buckets == 0 || q->n_columns == 0 || !q->columns) return TSKV_ERR_INVALID_ARG;
  uint64_t n_out = 0;
  for (uint32_t c = 0; c < q->n_columns; c++) n_out += popc(q->columns[c].agg_mask & TSKV_AGG_ALL);
  uint64_t n_groups = 1;
  if (q->group_by_series) {
    if (q->series_ids) {
      n_groups = q->n_series;
    } else {
      std::vector<uint32_t> ids;
      for (uint64_t i = 0; i < n_descs; i++)
        if (descs[i].phys_type == TSKV_PT_TIME) ids.push_back(descs[i].series_id);
      std::sort(ids.begin(), ids.end());
      n_groups = (uint64_t)(std::unique(ids.begin(), ids.end()) - ids.begin());
    }
  }
  out->n_out = n_out;
  out->n_groups = n_groups;
  out->n_cells = n_groups * q->n_buckets;
  out->bitmap_stride = (out->n_cells + 63) / 64 * 8;
  out->values_bytes = n_out * out->n_cells * 8;
  out->validity_bytes = n_out * out->bitmap_stride;
  return TSKV_OK;
}

tskv_status orc_scan_aggregate(const uint8_t *arena, uint64_t arena_len,
                               const tskv_page_desc *descs, uint64_t n_descs, const tskv_query *q,
                               int verify_crc, int n_threads, uint64_t *out_values,
                               uint8_t *out_validity, uint64_t *out_points) {
  return orc_scan_aggregate_tomb(arena, arena_len, descs, n_descs, q, nullptr, 0, verify_crc, n_threads, out_values,
                                 out_validity, out_points);
}

}  // extern "C"

namespace {

// An opened page set: the series index is built ONCE here, like the reference's cached TsmReader metadata
// (tskv/src/tsm/reader.rs:120-168 loaded on open, kept by the version's reader cache, tsfamily/version.rs:158-172),
// and a persistent pool of worker threads stands in for the tokio/rayon workers the reference keeps alive.
struct Pool {
  std::vector<std::thread> workers;
  std::mutex mu;
  std::condition_variable cv_go, cv_done;
  std::function<void(uint64_t)> job;
  uint64_t n_jobs = 0, next = 0, done = 0, epoch = 0;
  bool stop = false;
  explicit Pool(unsigned n) {
    for (unsigned i = 0; i < n; i++) workers.emplace_back([this]() { loop(); });
  }
  ~Pool() {
    {
      std::lock_guard<std::mutex> l(mu);
      stop = true;
    }
    cv_go.notify_all();
    for (auto &t : workers) t.join();
  }
  void loop() {
    uint64_t seen = 0;
    for (;;) {
      std::unique_lock<std::mutex> l(mu);
      cv_go.wait(l, [&]() { return stop || (epoch != seen && next < n_jobs); });
      if (stop) return;
      while (next < n_jobs) {
        uint64_t k = next++;
        l.unlock();
        job(k);
        l.lock();
        if (++done == n_jobs) cv_done.notify_all();
      }
      seen = epoch;
    }
  }
  void run(uint64_t n, std::function<void(uint64_t)> f) {
    std::unique_lock<std::mutex> l(mu);
    job = std::move(f);
    n_jobs = n;
    next = 0;
    done = 0;
    epoch++;
    cv_go.notify_all();
    cv_done.wait(l, [&]() { return done == n_jobs; });
  }
};

}  // namespace

struct orc_handle {
  const uint8_t *arena;
  uint64_t arena_len;
  const tskv_page_desc *descs;
  uint64_t n_descs;
  Index ix;
  int n_threads;
  Pool *pool;
  std::vector<std::vector<Cell>> priv;  // per-chunk partial tables, kept between scans
  std::vector<uint64_t> cg_file;         // orc_set_chunk_files
};

namespace {

tskv_status scan_with(orc_handle *H, const tskv_query *q, const tskv_tombstone *tombs, uint64_t n_tombs,
                      int verify_crc, uint64_t *out_values, uint8_t *out_validity, uint64_t *out_points);

}  // namespace

extern "C" {

tskv_status orc_open(const uint8_t *arena, uint64_t arena_len, const tskv_page_desc *descs, uint64_t n_descs,
                     int n_threads, orc_handle **out) {
  g_err.clear();
  if (!out) return TSKV_ERR_INVALID_ARG;
  orc_handle *H = new orc_handle{arena, arena_len, descs, n_descs, Index{}, n_threads, nullptr, {}, {}};
  tskv_status st = build_index(descs, n_descs, H->ix);
  if (st != TSKV_OK) {
    delete H;
    return st;
  }
  if (n_threads > 1) H->pool = new Pool((unsigned)n_threads);
  *out = H;
  return TSKV_OK;
}

// Tags every column group (descriptor-table order) with the id of the file its chunk belongs to: scans then group a
// series' chunks by time-range overlap and merge overlapping ones (reader/iterator.rs:463-560). n_cg == 0 clears.
tskv_status orc_set_chunk_files(orc_handle *H, const uint64_t *cg_file_id, uint64_t n_cg) {
  if (!H || (n_cg && !cg_file_id)) return TSKV_ERR_INVALID_ARG;
  if (n_cg == 0) {
    H->cg_file.clear();
    return TSKV_OK;
  }
  if (n_cg != H->ix.cgs.size()) {
    g_err = "one file id per column group expected";
    return TSKV_ERR_INVALID_ARG;
  }
  H->cg_file.assign(cg_file_id, cg_file_id + n_cg);
  std::vector<uint64_t> t;
  std::vector<uint8_t> tv;
  for (ColumnGroup &cg : H->ix.cgs) {
    const tskv_page_desc &td = H->descs[cg.first_desc];
    t.assign(td.num_values ? td.num_values : 1, 0);
    tv.assign(td.num_values ? td.num_values : 1, 0);
    uint64_t nr = 0;
    tskv_status st = orc_page_decode(TSKV_PT_TIME, H->arena + td.offset, td.size, 0, t.data(), tv.data(), td.num_values, &nr);
    if (st != TSKV_OK) return st;
    cg.min_ts = INT64_MAX;
    for (uint64_t r = 0; r < nr; r++)
      if (tv[r]) cg.min_ts = std::min(cg.min_ts, (int64_t)t[r]);
  }
  return TSKV_OK;
}

void orc_close(orc_handle *H) {
  if (!H) return;
  delete H->pool;
  delete H;
}

tskv_status orc_scan(orc_handle *H, const tskv_query *q, const tskv_tombstone *tombs, uint64_t n_tombs, int verify_crc,
                     uint64_t *out_values, uint8_t *out_validity, uint64_t *out_points) {
  if (!H) return TSKV_ERR_INVALID_ARG;
  return scan_with(H, q, tombs, n_tombs, verify_crc, out_values, out_validity, out_points);
}

tskv_status orc_scan_aggregate_tomb(const uint8_t *arena, uint64_t arena_len,
                                    const tskv_page_desc *descs, uint64_t n_descs, const tskv_query *q,
                                    const tskv_tombstone *tombs, uint64_t n_tombs,
                                    int verify_crc, int n_threads, uint64_t *out_values,
                                    uint8_t *out_validity, uint64_t *out_points) {
  orc_handle *H = nullptr;
  tskv_status st = orc_open(arena, arena_len, descs, n_descs, n_threads, &H);
  if (st != TSKV_OK) return st;
  st = orc_scan(H, q, tombs, n_tombs, verify_crc, out_values, out_validity, out_points);
  orc_close(H);
  return st;
}

}  // extern "C"

namespace {

tskv_status scan_with(orc_handle *H, const tskv_query *q, const tskv_tombstone *tombs, uint64_t n_tombs,
                      int verify_crc, uint64_t *out_values, uint8_t *out_validity, uint64_t *out_points) {
  g_err.clear();
  const tskv_page_desc *descs = H->descs;
  const uint64_t n_descs = H->n_descs;
  const Index &ix = H->ix;
  const int n_threads = H->n_threads;
  tskv_output_layout L;
  tskv_status st = orc_query_output_layout(descs, n_descs, q, &L);
  if (st != TSKV_OK) return st;
  Scan S{H->arena, H->arena_len, descs, q, verify_crc, &ix, {}, L.n_cells};
  S.tombs = tombs;
  S.n_tombs = n_tombs;
  S.cg_file = H->cg_file.empty() ? nullptr : H->cg_file.data();
  S.value_stats_pruning = g_value_stats_pruning;
  if (q->series_ids) {
    for (uint32_t i = 0; i < q->n_series; i++) {
      if (i && q->series_ids[i] <= q->series_ids[i - 1]) {
        g_err = "series_ids must be sorted ascending and unique";
        return TSKV_ERR_INVALID_ARG;
      }
    }
    S.slots.assign(q->series_ids, q->series_ids + q->n_series);
  } else {
    S.slots = ix.series;
  }
  uint64_t n_slots = S.slots.size();
  uint64_t table = (uint64_t)q->n_columns * L.n_cells;
  std::vector<Cell> cells(table);
  uint64_t points = 0;
  if (n_threads <= 1 || n_slots < 2 || !H->pool) {
    st = scan_slots(S, 0, n_slots, cells.data(), true, &points);
    if (st != TSKV_OK) return st;
  } else {
    // contiguous chunks of (n + ncpu) / ncpu series, like tskv/src/reader/iterator.rs:232-235
    uint64_t ncpu = (uint64_t)n_threads;
    uint64_t cs = (n_slots + ncpu) / ncpu;
    uint64_t n_chunks = (n_slots + cs - 1) / cs;
    std::vector<tskv_status> sts(n_chunks, TSKV_OK);
    std::vector<uint64_t> pts(n_chunks, 0);
    std::vector<std::string> errs(n_chunks);
    std::vector<std::vector<Cell>> &priv = H->priv;
    if (!q->group_by_series) {
      if (priv.size() < n_chunks) priv.resize(n_chunks);
      for (uint64_t k = 0; k < n_chunks; k++) priv[k].assign(table, Cell{});
    }
    H->pool->run(n_chunks, [&](uint64_t k) {
      g_err.clear();
      Cell *dst = q->group_by_series ? cells.data() : priv[k].data();  // disjoint cells per slot
      sts[k] = scan_slots(S, k * cs, std::min(n_slots, (k + 1) * cs), dst, false, &pts[k]);
      errs[k] = g_err;
    });
    for (uint64_t k = 0; k < n_chunks; k++) {
      if (sts[k] != TSKV_OK) {
        g_err = errs[k];
        return sts[k];
      }
      points += pts[k];
      if (!q->group_by_series)
        for (uint32_t c = 0; c < q->n_columns; c++)
          for (uint64_t i = 0; i < L.n_cells; i++)
            merge_cell(cells[(uint64_t)c * L.n_cells + i], priv[k][(uint64_t)c * L.n_cells + i],
                       q->columns[c].phys_type);
    }
  }
  if (out_points) *out_points = points;
  // finalize into the dense layout of include/tskv_gpu.h
  memset(out_validity, 0, L.validity_bytes);
  uint64_t j = 0;
  for (uint32_t c = 0; c < q->n_columns; c++) {
    const tskv_agg_column &qc = q->columns[c];
    for (unsigned bit = 0; bit < 7; bit++) {
      unsigned agg = 1u << bit;
      if (!(qc.agg_mask & agg)) continue;
      uint64_t *ov = out_values + j * L.n_cells;
      uint8_t *ob = out_validity + j * L.bitmap_stride;
      for (uint64_t i = 0; i < L.n_cells; i++) {
        const Cell &cell = cells[(uint64_t)c * L.n_cells + i];
        uint64_t v = 0;
        bool valid = false;
        switch (agg) {
          case TSKV_AGG_COUNT:
            v = cell.count;
            valid = true;
            break;
          case TSKV_AGG_SUM:
            valid = cell.count > 0;
            if (valid) {
              if (qc.phys_type == TSKV_PT_F64)
                memcpy(&v, &cell.sum_d, 8);
              else
                v = cell.sum_bits;
            }
            break;
          case TSKV_AGG_MIN:
            valid = cell.count > 0;
            if (valid) v = cell.minv;
            break;
          case TSKV_AGG_MAX:
            valid = cell.count > 0;
            if (valid) v = cell.maxv;
            break;
          case TSKV_AGG_MEAN:
            valid = cell.count > 0;
            if (valid) {
              double m = cell.sum_d / (double)cell.count;
              memcpy(&v, &m, 8);
            }
            break;
          case TSKV_AGG_FIRST:
            valid = cell.has_first;
            if (valid) v = cell.first_val;
            break;
          case TSKV_AGG_LAST:
            valid = cell.has_last;
            if (valid) v = cell.last_val;
            break;
        }
        ov[i] = v;
        if (valid) ob[i >> 3] |= (uint8_t)(1u << (i & 7));
      }
      j++;
    }
  }
  return TSKV_OK;
}

}  // namespace
