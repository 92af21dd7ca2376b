/*
 * tskv_gpu.h — C ABI of the H100-native tskv scan/aggregate engine.
 *
 * This is the drop-in boundary for ONE path of cnosdb/cnosdb (all citations are relative to the
 * reference tree): TSM page decode -> time-range + series-selection filter -> time-bucketed
 * aggregate. The reference has no FFI; the seam it replaces is the `BatchReader` tree built by
 * `SeriesGroupBatchReaderFactory::create` (tskv/src/reader/iterator.rs:123-264) and polled through
 * `BatchReader::process` (tskv/src/reader/mod.rs:159-164). A Rust shim implementing that trait
 * binds the functions below (see INTEGRATION.md for the `extern "C"` block a maintainer would add).
 *
 * Conventions
 *   - plain C, no torch / CUDA types in any signature; device memory is addressed as uint64_t.
 *   - every entry point returns a tskv_status (0 = ok); nothing throws or aborts across the ABI.
 *   - the caller owns every host buffer it passes; the library copies and never frees them.
 *   - a context is bound to one CUDA device; calls on one context are serialised internally
 *     (thread-safe), different contexts are independent (one per tokio blocking thread / per GPU).
 */
#ifndef TSKV_GPU_H_
#define TSKV_GPU_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ------------------------------------------------------------------------------------------- */
/* Status codes. The decode codes map 1:1 onto the reference's codec error strings, which the   */
/* Rust side surfaces as TskvError::Decode (tskv/src/error.rs:293-299).                         */
/* ------------------------------------------------------------------------------------------- */
typedef int32_t tskv_status;
enum {
  TSKV_OK = 0,
  TSKV_ERR_INVALID_ARG = 1,     /* null pointer, malformed descriptor table, unsorted selection */
  TSKV_ERR_BAD_ENCODING = 2,    /* "invalid block encoding" (timestamp.rs:197, integer.rs:161) */
  TSKV_ERR_SHORT_BLOCK = 3,     /* "not enough data to decode ..." / "unexpected end of block"
                                   (timestamp.rs:228,263; integer.rs:188,218; float.rs:462) */
  TSKV_ERR_CRC_MISMATCH = 4,    /* TsmPageFileHashCheckFailed (tskv/src/tsm/page.rs:58-76) */
  TSKV_ERR_BITSET_MISMATCH = 5, /* "Mismatch between bit set and decoded values" (float.rs:598);
                                   also: fewer decoded values than valid bits in ts/i64 pages,
                                   which the reference turns into an Arrow length error */
  TSKV_ERR_UNSUPPORTED = 6,     /* Quantile(pco)/bool/string pages, or a first/last key that does
                                   not fit 63 bits (see DESIGN.md) */
  TSKV_ERR_BUCKET_RANGE = 7,    /* an in-range row fell outside [first_bucket_start, +n*width) */
  TSKV_ERR_CUDA = 8,
  TSKV_ERR_NCCL = 9,            /* an NCCL call failed, or libnccl could not be loaded (tskvgpu_comm_*) */
  TSKV_ERR_OOM = 10,
  TSKV_ERR_BAD_LENGTH = 11,     /* "invalid uncompressed block length" (timestamp.rs:203) */
  TSKV_ERR_PAGE_FORMAT = 12     /* page shorter than its own header / bitset (page.rs:78-94) */
};

/* Physical column type of a page: PhysicalCType::Time / PhysicalDType::{Integer,Unsigned,Float,Boolean}
 * (dispatch in tskv/src/tsm/reader.rs:658-731). Boolean pages (tskv/src/tsm/codec/boolean.rs:79-140: bit-packed, or one
 * byte per value under Encoding::Null) decode to 0 / 1 in the 8-byte cells; aggregates on them: count, min, max, first,
 * last (SUM / MEAN of a boolean column are rejected like DataFusion's type check does). String pages are not handled. */
enum {
  TSKV_PT_TIME = 0,
  TSKV_PT_I64 = 1,
  TSKV_PT_U64 = 2,
  TSKV_PT_F64 = 3,
  TSKV_PT_BOOL = 4
};

/* Encoding ids stored in data[0] of a page (common/models/src/codec.rs:37-54). */
enum {
  TSKV_ENC_DEFAULT = 0,
  TSKV_ENC_NULL = 1,
  TSKV_ENC_DELTA = 2,
  TSKV_ENC_QUANTILE = 3,
  TSKV_ENC_GORILLA = 6,
  TSKV_ENC_BITPACK = 10,
  TSKV_ENC_DELTA_TS = 11
};

/* One encoded page inside the arena. Replaces `PageWriteSpec{offset,size,meta}`
 * (tskv/src/tsm/page.rs:599-620) + the `Page.bytes` it addresses (page.rs:31-39).
 * Pages are listed column group by column group (tskv/src/tsm/column_group.rs:9-17): a TIME page
 * opens a column group and is followed by that group's field pages (ascending column id,
 * mem_cache/series_data.rs:226-230). All pages of a group carry the same series_id / num_values.
 * `offset` must be 16-byte aligned inside the arena. 24 bytes. */
typedef struct tskv_page_desc {
  uint64_t offset;     /* byte offset of the page (header+bitset+data) in the arena */
  uint32_t size;       /* page size in bytes */
  uint32_t num_values; /* PageMeta.num_values = rows incl. nulls (page.rs:347-351) */
  uint32_t series_id;  /* SeriesId (common/models/src/lib.rs:40), local to the vnode */
  uint16_t column_id;  /* TableColumn.id; ignored for the time page */
  uint8_t phys_type;   /* TSKV_PT_* */
  uint8_t reserved;    /* must be 0 (the library stores its decode-kind here on the device) */
} tskv_page_desc;

/* Closed interval, exactly `TimeRange{min_ts,max_ts}` (common/models/src/predicate/domain.rs:35-98). */
typedef struct tskv_time_range {
  int64_t min_ts;
  int64_t max_ts;
} tskv_time_range;

/* Aggregate bits. count/sum/min/max/avg follow DataFusion's builtins; first/last follow
 * query_server/query/src/extension/expr/aggregate_function/{first,last}.rs. */
enum {
  TSKV_AGG_COUNT = 1u << 0, /* valid (non-null) values in range; u64 */
  TSKV_AGG_SUM = 1u << 1,   /* i64/u64: wrapping; f64: double */
  TSKV_AGG_MIN = 1u << 2,
  TSKV_AGG_MAX = 1u << 3,
  TSKV_AGG_MEAN = 1u << 4,  /* f64 = sum / count */
  TSKV_AGG_FIRST = 1u << 5, /* value at the smallest timestamp */
  TSKV_AGG_LAST = 1u << 6,  /* value at the largest timestamp */
  TSKV_AGG_ALL = 0x7f,      /* the seven aggregates above (not M2) */
  /* f64 M2 = sum over the cell's valid, selected values of (x - mean)^2, x converted to f64 first (DataFusion's variance
   * state, with count: var_pop = M2 / n, var_samp = M2 / (n - 1), stddev* = sqrt(var*)). Valid iff the cell holds at least
   * one value; a one-value cell reads 0.0; NaN or +-inf among the values gives NaN. I64 / U64 / F64 columns; a BOOL column
   * is refused like SUM (TSKV_ERR_INVALID_ARG). Computed in two passes over the column's pages: pass 1 (the scan as
   * without M2, which also keeps the column's COUNT and exact SUM) gives every cell's mean m, pass 2 decodes the same rows
   * again and sums d = x - m and d^2; M2 = sum(d^2) - sum(d)^2 / n (corrected two-pass algorithm). Refused before any
   * launch with TSKV_ERR_UNSUPPORTED: sliding windows (slide != width). tskvgpu_scan_partials refuses a scan with M2.
   * Counters: page_read_count, page_read_bytes, points_decoded and rows_in_range are those of the same query without M2
   * (the reference reads each page once); kernel_launches and elapsed_fused_ms include pass 2. */
  TSKV_AGG_M2 = 1u << 7
};

/* One projected value column and the aggregates wanted for it. Extends
 * `PushedAggregateFunction` (common/models/src/predicate/domain.rs:1840-1843), which today only
 * has Count(col). */
typedef struct tskv_agg_column {
  uint16_t column_id;
  uint8_t phys_type; /* TSKV_PT_I64 / U64 / F64 / BOOL: pages of another type under this id are an error */
  uint8_t agg_mask;  /* TSKV_AGG_* bits */
} tskv_agg_column;

/* A field-value comparison pushed into the scan (the row filter of DataFilter, tskv/src/reader/filter.rs:23-142, for
 * predicates of the form `column <op> constant` joined by AND): a row is kept only if EVERY predicate is TRUE for it.
 * A NULL value - or a column group that holds no page of the column, which the reference null-fills
 * (reader/schema_alignmenter.rs:24-44) - makes the comparison NULL, and filter_record_batch drops the row like a FALSE.
 * Dropped rows count for no projected column (count, sum, first/last ...), exactly like rows outside the time ranges.
 * Integers compare as their type, f64 numerically (NaN: never TRUE; the reference's arrow kernels are not pinned for
 * NaN / signed zeros inside the reference tree). `value` holds the constant's bit pattern.
 * Column groups in which the min / max of a predicate column's page rule the comparison out for every row are not read at
 * all (filter_column_groups with PageMeta.statistics, tskv/src/reader/chunk.rs:12-50; the statistics are computed on the
 * device once per HBM-resident page set); tskv_counters.pruned_page_count counts their pages. */
enum { TSKV_CMP_EQ = 0, TSKV_CMP_NE = 1, TSKV_CMP_LT = 2, TSKV_CMP_LE = 3, TSKV_CMP_GT = 4, TSKV_CMP_GE = 5 };
#define TSKV_MAX_PREDICATES 8
typedef struct tskv_field_predicate {
  uint16_t column_id;
  uint8_t phys_type; /* TSKV_PT_I64 / U64 / F64 */
  uint8_t op;        /* TSKV_CMP_* */
  uint32_t reserved;
  uint64_t value;
} tskv_field_predicate;

/* The pushed-down scan. Mirrors the fields of `QueryOption` the hot path consumes
 * (tskv/src/reader/iterator.rs:713-741): split.time_ranges(), the series ids produced by
 * `get_series_id_by_filter` (tskv/src/kvcore.rs:249-279), the aggregate list; plus the bucket
 * expression `time_window(time, width)` / `date_bin(width, time, origin)` that today runs in
 * DataFusion (query_server/query/src/extension/analyse/transform_time_window.rs:251-296). */
typedef struct tskv_query {
  const uint32_t *series_ids; /* sorted ascending, unique; NULL => every series of the arena.
                                 The position of an id in this list is its "slot": it is the
                                 group index when group_by_series != 0 and the tie-break order of
                                 first/last ("earlier-seen point wins", first.rs:103-107). */
  uint32_t n_series;
  uint32_t n_time_ranges; /* 0 => all time */
  const tskv_time_range *time_ranges;
  int64_t origin;             /* start_time of the window expression */
  int64_t width;              /* bucket width in the time column's unit; <= 0 => no bucketing */
  int64_t first_bucket_start; /* start of output bucket 0 (must be a value the formula yields) */
  uint32_t n_buckets;         /* >= 1 (1 when width <= 0) */
  uint32_t group_by_series;   /* 0: GROUP BY bucket ; 1: GROUP BY series, bucket */
  const tskv_agg_column *columns;
  uint32_t n_columns;         /* 1..126 */
  uint32_t reserved;          /* TSKV_QUERY_* flags (0 for a plain single-device scan) */
  const tskv_field_predicate *predicates; /* AND-ed field comparisons, or NULL */
  uint32_t n_predicates;      /* 0..TSKV_MAX_PREDICATES */
  uint32_t n_pairs;           /* 0..TSKV_MAX_PAIRS column pairs (covariance / correlation state, below); 0: none */
} tskv_query;
/* Column pairs: covar / covar_samp / covar_pop / corr (DataFusion's Covariance / Correlation). The 2 * n_pairs entries of
 * `columns` after the n_columns projected ones are the pairs' operands x0, y0, x1, y1, ...: column_id and phys_type
 * (I64 / U64 / F64) of each, agg_mask 0. n_columns may be 0 when n_pairs >= 1; n_columns + 2 * n_pairs <= 126; x may equal
 * y. Both operands convert to f64. A row counts for a pair when it is selected (time ranges, series, the row filter of
 * the predicates, row-drop tombstones) and both x and y are valid (non-NULL after column tombstones); a column group
 * without a page of x or of y has no paired row. Per cell each pair adds four outputs after every column output, in pair
 * order: n (u64, the paired rows, valid like COUNT), then f64 C = sum (x - mx)(y - my), M2x = sum (x - mx)^2 and
 * M2y = sum (y - my)^2 over the paired rows (mx, my: their paired means), valid iff n >= 1. M2x is exactly 0.0 when the
 * paired x values are all equal and finite (M2y alike); NaN or +-inf among them gives NaN. The host derives
 * covar = covar_samp = C / (n - 1), covar_pop = C / n, corr = (C / n) / sqrt(M2x / n) / sqrt(M2y / n) (0.0 when either
 * root is 0). Computed in two passes over the rows of x's pages paired with the same column group's y page: pass 1 sums
 * n, x and y per cell, pass 2 sums dx = x - sum x / n, dy, dx dy, dx^2 and dy^2; C = sum dx dy - sum dx sum dy / n,
 * M2 = sum d^2 - (sum d)^2 / n (corrected two-pass algorithm). An operand that is not a projected column is read like a
 * COUNT column that has no output. Refused before any launch: TSKV_ERR_INVALID_ARG for n_pairs > TSKV_MAX_PAIRS, an
 * operand with a non-zero agg_mask or a BOOL / TIME / unknown type, an operand id projected with another type, or more
 * than 126 columns; TSKV_ERR_UNSUPPORTED for sliding windows (slide != width). tskvgpu_scan_partials refuses a scan with
 * pairs (use tskvgpu_scan_exchange / _merge_gathered, which merge the ranks' co-moments with Chan's formula). Pages of
 * another type under an operand's id are an error. Counters: page_read_count, page_read_bytes, points_decoded,
 * rows_in_range and pruned_page_count equal those of the same query with every operand that is not projected added as a
 * COUNT column; kernel_launches and elapsed_fused_ms include the pair passes. */
#define TSKV_MAX_PAIRS 8
/* The partial state of this scan will be merged with other ranks' (tskvgpu_scan_partials / _exchange_view): every
 * exchanged key is then derived from the query alone, never from this rank's own arena (its time bounds, its local
 * series ranks), so that all ranks build comparable first/last tie-break keys. Requires series_ids != NULL when the
 * query groups by series or asks for first/last; unbucketed first/last across series need bounded time ranges. */
#define TSKV_QUERY_MULTI_RANK 1u
/* Medians: median(x) (DataFusion's MedianAccumulator), exact. Bits 8..15 of the flags word (`reserved`) hold n_medians:
 * TSKV_QUERY_MEDIANS(n) sets them, TSKV_QUERY_N_MEDIANS(flags) reads them. The n_medians entries of `columns` after the
 * pairs' 2 * n_pairs operands are the medians' operands: column_id and phys_type (I64 / U64 / F64) of each, agg_mask 0;
 * n_columns may be 0; n_columns + 2 * n_pairs + n_medians <= 126. A median takes the operand's values in the selected rows
 * (time ranges, series, the row filter of the predicates, row-drop and column tombstones), NULLs left out, ordered by the
 * type's order (f64: IEEE totalOrder; NaN is a value). Per cell each median adds one output after the pairs' outputs, in
 * the operand's type, valid iff the cell holds a value: for odd n the value at rank n / 2 (from 0), for even n
 * (lo + hi) / 2 of the values lo, hi at ranks n / 2 - 1 and n / 2 in the operand's type: i64 wrapping add, then division
 * truncating toward zero; u64 wrapping add, then / 2; f64 (lo + hi) / 2.0 with x86-64 NaN results (a NaN operand's bits,
 * quieted, lo first; -inf + inf gives 0xfff8000000000000). Computed by radix selection on the order keys: pass 1 gives
 * every cell's n and extreme keys (the operand's kernel mask gains COUNT | MIN | MAX; an operand that is not a projected
 * column is read like such a column with no output), then 8 selection passes over the operand's pages each narrow the
 * keys at the two ranks by an 8-bit digit (histograms of 1 KiB per cell and median) until a cell is resolved; passes
 * that no cell needs decode nothing. Refused before any launch: TSKV_ERR_INVALID_ARG for n_medians > TSKV_MAX_MEDIANS, an
 * operand with a non-zero agg_mask or a BOOL / TIME / unknown type, an operand id projected with another type, or more
 * than 126 columns; TSKV_ERR_UNSUPPORTED for sliding windows (slide != width), TSKV_QUERY_MULTI_RANK, more than
 * TSKV_MAX_MEDIAN_CELLS cells times medians (the histogram budget, 4 GiB; GROUP BY series over 100 000 series x 168
 * buckets exceeds it), and an operand whose pages hold 2^32 rows or more (the histograms count in 32 bits).
 * tskvgpu_scan_partials, _exchange_view, _exchange and _merge_gathered refuse a scan with medians. Pages of another type
 * under an operand's id are an error. Counters: page_read_count, page_read_bytes, points_decoded, rows_in_range and
 * pruned_page_count equal those of the same query with every operand that is not projected added as a COUNT column;
 * kernel_launches and elapsed_fused_ms include the selection passes. */
#define TSKV_MAX_MEDIANS 8
#define TSKV_MAX_MEDIAN_CELLS (1u << 22)
#define TSKV_QUERY_MEDIANS(n) (((uint32_t)(n) & 0xffu) << 8)
#define TSKV_QUERY_N_MEDIANS(flags) (((uint32_t)(flags) >> 8) & 0xffu)
/* Counter increases: increase(time, x ORDER BY time) (CnosDB's IncreaseAccumulator). Bits 16..23 of the flags word hold
 * n_increases: TSKV_QUERY_INCREASES(n) sets them, TSKV_QUERY_N_INCREASES(flags) reads them. The n_increases entries of
 * `columns` after the medians' operands are the increases' operands: column_id and phys_type (I64 / U64 / F64) of each,
 * agg_mask 0; n_columns + 2 * n_pairs + n_medians + n_increases <= 126. An increase walks a cell's selected rows (time
 * ranges, series, the row filter of the predicates, row-drop and column tombstones, non-NULL time) in time order, NULL
 * operand values left out; each value v after the previous one `last` adds v - last when v > last, v when v < last (a
 * counter reset) and nothing when they are equal; the sum starts at 0. Integers subtract and sum wrapping (i64 compares
 * signed, u64 unsigned); f64 compares by IEEE totalOrder and sums in atomic order. Per cell each increase adds one output
 * after the medians' outputs, in the operand's type, valid iff the cell holds a value of the operand (the reference
 * prints 0 for a group whose operand is NULL in every row). A cell must hold rows of one series only: the scan runs the
 * operand as a COUNT column in pass 1, then one lane per page pairs consecutive rows and records the page's first and
 * last selected points, every merged row of the overlap merge groups is a record of its own, and the records of every
 * series, sorted by time, add the pairs across their boundaries. The increases sit in the exchange
 * region's integer / f64 sum sections: tskvgpu_scan_partials, _exchange and _merge_gathered sum them across ranks.
 * Refused before any launch: TSKV_ERR_INVALID_ARG for n_increases > TSKV_MAX_INCREASES, an operand with a non-zero agg_mask
 * or a BOOL / TIME / unknown type, an operand id projected with another type, or more than 126 columns;
 * TSKV_ERR_UNSUPPORTED for a cell that could hold rows of two selected series (an ungrouped scan over more than one
 * selected series - series_ids NULL: the page set holds more than one; with TSKV_QUERY_MULTI_RANK, series_ids NULL at
 * all, so that every rank decides from the query alone - or a group map with two selected slots in one group), sliding windows (slide != width) and tskvgpu_scan_prepare_labels. Counters: as for medians; kernel_launches and
 * elapsed_fused_ms include the increase kernels. */
#define TSKV_MAX_INCREASES 8
#define TSKV_QUERY_INCREASES(n) (((uint32_t)(n) & 0xffu) << 16)
#define TSKV_QUERY_N_INCREASES(flags) (((uint32_t)(flags) >> 16) & 0xffu)

/* Result layout. Outputs are dense: for output column j (query columns in order, and inside a
 * column the set agg bits in ascending bit order) and cell c = group * n_buckets + bucket:
 *   values  [j * n_cells + c]                     8-byte cell (i64 / u64 / f64 bit pattern)
 *   validity[j * bitmap_stride + (c >> 3)] bit (c & 7)   Arrow LSB-first validity
 * so a shim can wrap each output column zero-copy as an Arrow array. */
typedef struct tskv_output_layout {
  uint64_t n_out;         /* number of output columns */
  uint64_t n_groups;      /* 1, number of series slots when group_by_series, or n_groups of a *_grouped call */
  uint64_t n_cells;       /* n_groups * n_buckets */
  uint64_t bitmap_stride; /* bytes per validity bitmap, multiple of 8 */
  uint64_t values_bytes;  /* n_out * n_cells * 8 */
  uint64_t validity_bytes;/* n_out * bitmap_stride */
} tskv_output_layout;

/* Counters mirroring the reference's per-operator metrics (reader/column_group/mod.rs:141-193:
 * page_read_count, page_read_bytes, elapsed_page_scan_time, elapsed_page_to_array_time). */
typedef struct tskv_counters {
  uint64_t page_read_count;     /* pages touched by the last scan */
  uint64_t page_read_bytes;     /* encoded bytes of those pages (algorithmic bytes numerator) */
  uint64_t points_decoded;      /* valid values decoded by the last scan/decode */
  uint64_t rows_in_range;       /* rows that passed the time filter */
  double elapsed_scan_ms;       /* device time of the last scan (CUDA events) */
  double elapsed_h2d_ms;        /* host->device time of the last upload / query arguments */
  uint64_t kernel_launches;     /* kernels launched by the last call */
  double elapsed_fused_ms;      /* device time of the fused decode/filter/reduce kernels alone */
  double dominant_kernel_ms;    /* slowest fused kernel (one per decode-kind bin) of the last scan */
  uint64_t dominant_kernel_bytes; /* encoded page bytes that kernel read (its algorithmic bytes) */
  uint64_t dominant_kernel_bin; /* 0-8: time-codec class * 3 + value-codec class; 9-12: the short-page bins
                                   (pages of <= 1024 rows, see DESIGN.md) */
  uint64_t h2d_bytes;           /* query arguments copied host->device by the last prepare */
  uint64_t pruned_page_count;   /* selected field pages the last scan skipped because their column group's time bounds
                                   miss every query range (filter_column_groups, reader/chunk.rs:12-50) */
} tskv_counters;

typedef struct tskv_ctx tskv_ctx;       /* one CUDA device + stream */
typedef struct tskv_pages tskv_pages;   /* a device-resident page arena + descriptor tables */

/* ---- context ------------------------------------------------------------------------------ */
tskv_status tskvgpu_ctx_create(int32_t device_id, tskv_ctx **out_ctx);
void tskvgpu_ctx_destroy(tskv_ctx *ctx);
/* Last error message of this context (valid until the next call on it). */
const char *tskvgpu_last_error(const tskv_ctx *ctx);
/* Index of the page that caused the last decode error, or -1. */
int64_t tskvgpu_last_error_page(const tskv_ctx *ctx);
tskv_status tskvgpu_get_counters(const tskv_ctx *ctx, tskv_counters *out);
/* Raw cudaStream_t of the context (as an integer) so a host runtime can order its own
 * collectives after a scan. */
uint64_t tskvgpu_ctx_stream(const tskv_ctx *ctx);

/* ---- pages ---------------------------------------------------------------------------------
 * Replaces TsmReader::read_adjacent_pages + Page::crc_validation (tskv/src/tsm/reader.rs:236-264,
 * page.rs:58-76): copies `arena` to the device, validates framing, optionally verifies each
 * page's CRC32 (flags & TSKV_UPLOAD_VERIFY_CRC) like the reference does on every read. */
enum {
  TSKV_UPLOAD_VERIFY_CRC = 1u,
  /* Keep the page bytes in the caller's host memory (page-locked by the library; the caller must keep
   * `arena` alive and unchanged until tskvgpu_pages_destroy) and let every scan pull only the
   * selected pages over PCIe — the analogue of the reference reading pages of the selected series
   * from the page cache on each query. Descriptor tables still live on the device (TsmReader
   * metadata is cached in the reference too: tsfamily/version.rs:158-172). Combined with
   * TSKV_UPLOAD_VERIFY_CRC the CRC32 of every page a scan reads is re-checked on the device after the
   * transfer, i.e. on every read like Page::crc_validation (tsm/reader.rs:259,492). */
  TSKV_UPLOAD_HOST_RESIDENT = 2u,
  /* Re-check the CRC32 of every page a scan reads on the device, on every scan, also for a device-resident arena
   * (host-resident + VERIFY_CRC page sets always do): the reference validates a page's CRC on each read
   * (tsm/reader.rs:259,492), not once per file. */
  TSKV_UPLOAD_VERIFY_ON_READ = 4u
};
tskv_status tskvgpu_upload_pages(tskv_ctx *ctx, const uint8_t *arena, uint64_t arena_len,
                                 const tskv_page_desc *descs, uint64_t n_descs, uint32_t flags,
                                 tskv_pages **out_pages);
void tskvgpu_pages_destroy(tskv_ctx *ctx, tskv_pages *pages);
/* Number of distinct series in the arena. */
uint64_t tskvgpu_pages_series_count(const tskv_pages *pages);
/* Per-column-group time bounds, `ColumnGroup::time_range()` (tskv/src/tsm/column_group.rs:9-17), in descriptor order
 * (one entry per TIME page; n must equal the number of column groups). Optional: scans with time ranges use them to
 * skip whole column groups (statistics pruning, reader/chunk.rs:12-50 + column_group/statistics.rs:11-80); a page set
 * without them gets its bounds from one device pass over the time pages on the first scan that needs them. */
tskv_status tskvgpu_pages_set_time_bounds(tskv_ctx *ctx, tskv_pages *pages, const tskv_time_range *bounds, uint64_t n);

/* ---- tombstones ------------------------------------------------------------------------------
 * Replaces the tombstone half of decode_pages (tskv/src/tsm/reader.rs:507-551,634-656) with the
 * TsmTombstone cache as its source (tsm/tombstone.rs:417-550). One entry = one closed time range:
 *   series_id = s, column_id = c      rows of (s, c) whose time lies in the range read as NULL
 *                                     (column_excluded: update_nullbits_by_time_range + updated_nullbuffer)
 *   series_id = TSKV_TOMB_ALL         the range is in the file's `all_excluded` set: those ROWS are dropped
 *     (column_id = TSKV_TOMB_ALL)     for every series of this page set (filter_record_batch, reader.rs:546-550)
 *   series_id = s, column_id = TSKV_TOMB_ALL   same, scoped to one series (for page sets assembled from
 *                                     several TSM files, whose `all_excluded` sets differ)
 * The reference locates the rows with a binary search over the page's time values; time pages are strictly
 * increasing (tsm/chunk.rs:100-110), for which that equals the row-wise test min_ts <= t <= max_ts used here.
 * The call replaces the page set's previous tombstones (n = 0 clears them) and must not overlap a scan
 * of the same page set. Tombstones apply to scans; tskvgpu_decode_pages stays Page::to_arrow_array. */
#define TSKV_TOMB_ALL 0xffffffffu
typedef struct tskv_tombstone {
  uint32_t series_id;
  uint32_t column_id;
  int64_t min_ts, max_ts; /* closed */
} tskv_tombstone;
tskv_status tskvgpu_pages_set_tombstones(tskv_ctx *ctx, tskv_pages *pages, const tskv_tombstone *tombs,
                                         uint64_t n_tombs);

/* Value statistics of the pages, handed in by the caller: PageMeta.statistics (tskv/src/tsm/page.rs:599-613,
 * tskv/src/tsm/statistics/mod.rs:4-9; what `tskvtsm_load` reports). stats[i] belongs to descriptor i (time pages: ignored).
 * With TSKV_STATS_MINMAX set, every non-null value of the page lies in [min, max] (bit patterns of the page's physical
 * type; bounds may be loose; min > max = the page holds no value); without it nothing is known about the page.
 * Scans with field predicates then skip the column groups the bounds rule out (filter_column_groups,
 * tskv/src/reader/chunk.rs:12-50) - also for TSKV_UPLOAD_HOST_RESIDENT page sets, whose pages the library never reads
 * ahead of a scan. Without this call, HBM-resident page sets compute exact statistics on the device on first use.
 * f64 bounds that are NaN are treated as unknown. n_descs must equal the page set's descriptor count. */
#define TSKV_STATS_MINMAX 1u
typedef struct tskv_value_stats {
  uint64_t min, max;
  uint32_t flags;
  uint32_t reserved;
} tskv_value_stats;
tskv_status tskvgpu_pages_set_value_stats(tskv_ctx *ctx, tskv_pages *pages, const tskv_value_stats *stats, uint64_t n_descs);

/* Overlapping chunks. A page set may hold the column groups of SEVERAL files (TSM files, delta files) and of the
 * memcache (its row groups handed in as raw-encoded pages): cg_file_id[k] is the id of the file column group k (in
 * descriptor-table order) came from - ColumnFile::file_id() / the cache's file id. Replaces, for later scans,
 *   build_series_reader: chunks sorted by time range, group_overlapping_segments, groups sorted by file id
 *                        (tskv/src/reader/iterator.rs:463-560, tskv/src/reader/utils.rs:77-107)
 *   DataMerger / sort_merge / BatchMergeBuilder: k-way merge on `time`, ties to the lower stream; rows with equal
 *                        time collapse, every column taking the last non-null value (tskv/src/reader/merge.rs,
 *                        sort_merge.rs:153-400, batch_builder.rs:74-155)
 *   MemCacheReader       (tskv/src/reader/memcache_reader.rs:33-165): the cache is one more chunk.
 * Chunks of a series whose time ranges do not overlap are scanned as before. The column groups' time bounds are
 * taken from tskvgpu_pages_set_time_bounds when it was called BEFORE this call, else computed from the time pages (bounds
 * handed in later do not regroup the chunks: call this again). n_cg = 0 clears;
 * any change invalidates scans prepared earlier (TSKV_ERR_INVALID_ARG when run). Time pages of overlapping chunks
 * must not hold NULLs (TSKV_ERR_UNSUPPORTED; the reference's writer never produces them). The merged rows of one
 * overlap group count as ONE record batch for first / last (the reference cuts batches of QueryOption.batch_size). */
tskv_status tskvgpu_pages_set_chunk_files(tskv_ctx *ctx, tskv_pages *pages, const uint64_t *cg_file_id, uint64_t n_cg);

/* ---- decode only ---------------------------------------------------------------------------
 * Replaces Page::to_arrow_array / data_buf_to_arrow_array (tskv/src/tsm/reader.rs:658-731) for
 * pages [first_page, first_page + n_pages): row r of page p lands at out_values[row_offsets[p]+r]
 * where row_offsets is the exclusive prefix sum of num_values over the requested pages; validity
 * is one Arrow LSB-first bitmap per page, page p starting at byte validity_offsets[p] =
 * sum over previous pages of ((num_values + 63) / 64) * 8. Null rows hold 0. Host buffers. */
tskv_status tskvgpu_decode_pages(tskv_ctx *ctx, const tskv_pages *pages, uint64_t first_page,
                                 uint64_t n_pages, uint64_t *out_values, uint8_t *out_validity);

/* ---- scan + filter + bucket aggregate ------------------------------------------------------ */
tskv_status tskvgpu_query_output_layout(const tskv_pages *pages, const tskv_query *q,
                                        tskv_output_layout *out);
/* Fused decode -> filter -> bucket reduce. `out_values` / `out_validity` are HOST buffers sized by
 * tskvgpu_query_output_layout (query arguments go host->device and results device->host inside
 * this call: this is the end-to-end path a BatchReader::process() would take). */
tskv_status tskvgpu_scan_aggregate(tskv_ctx *ctx, const tskv_pages *pages, const tskv_query *q,
                                   uint64_t *out_values, uint8_t *out_validity);

/* Device-resident variant used for multi-GPU partial reduction and for kernel-only timing:
 *   prepare  : uploads the query (selection list, ranges), builds the compacted work list and
 *              allocates the partial-aggregate state on the device.
 *   run      : zeroes the state and runs the fused kernel (no host<->device traffic).
 *   partials : exposes the raw state as four device sections a host runtime can all-reduce
 *              element-wise (i64 SUM / f64 SUM / i64 MIN / i64 MAX; see DESIGN.md "Multi-GPU").
 *   finalize : turns the (possibly all-reduced) state into the dense result and copies it to
 *              the host buffers. */
typedef struct tskv_scan tskv_scan;
typedef struct tskv_partials_view {
  uint64_t sum_i64_ptr, sum_i64_len; /* counts, i64/u64 sums          : all-reduce SUM as int64 */
  uint64_t sum_f64_ptr, sum_f64_len; /* f64 sums                      : all-reduce SUM as float64 */
  uint64_t min_i64_ptr, min_i64_len; /* ordered keys of MIN and FIRST : all-reduce MIN as int64 */
  uint64_t max_i64_ptr, max_i64_len; /* ordered keys of MAX and LAST  : all-reduce MAX as int64 */
  uint64_t sel_val_ptr, sel_val_len; /* FIRST then LAST values, same order as their keys; after
                                        the key all-reduce call tskvgpu_scan_mask_values and
                                        all-reduce SUM this section as int64 */
  uint64_t sel_first_len;            /* number of FIRST cells (prefix of sel_val / suffix of min) */
  uint64_t sel_last_len;             /* number of LAST cells */
} tskv_partials_view;
/* A scan with TSKV_AGG_M2 has no partials view (TSKV_ERR_UNSUPPORTED): second moments taken around each rank's own means
 * do not all-reduce element-wise. Its ranks merge with tskvgpu_scan_exchange / _merge_gathered, which combine the ranks'
 * (count, sum, M2) with Chan's formula M2 = sum M2_r + sum n_r (m_r - m)^2. */

tskv_status tskvgpu_scan_prepare(tskv_ctx *ctx, const tskv_pages *pages, const tskv_query *q,
                                 tskv_scan **out_scan);
tskv_status tskvgpu_scan_run(tskv_ctx *ctx, tskv_scan *scan);
/* scan_run == scan_enqueue (launches only, no host synchronisation; safe to call repeatedly) followed
 * by scan_sync (waits, reports device-side decode errors, refreshes the counters). */
tskv_status tskvgpu_scan_enqueue(tskv_ctx *ctx, tskv_scan *scan);
tskv_status tskvgpu_scan_sync(tskv_ctx *ctx, tskv_scan *scan);
tskv_status tskvgpu_scan_partials(tskv_ctx *ctx, tskv_scan *scan, tskv_partials_view *out);
/* The work list of the scan's last pass (after scan_run / scan_sync), for tests and diagnostics. Bucket
 * k = (bin * n_columns + column) * 2 + narrow flag owns the items [region_start[k], region_start[k] + fill[k]).
 * Outputs (each may be null): region_start [n_buckets + 1], fill [n_buckets], work_page / work_slot [n_items],
 * work_qcol [n_items] (query column | 0x80 when the item brings its column group's time page), and per descriptor of
 * the page set page_bin / page_narrow [n_descs] (decode-kind bin and narrow flag of a field page, what the walk keys
 * its buckets on; page_narrow is all 0 when the scan does not keep narrow pages apart). *n_buckets and *n_items
 * (= region_start[n_buckets]) are always written: call with null arrays first to size them. */
tskv_status tskvgpu_scan_work_list(tskv_ctx *ctx, tskv_scan *scan, uint32_t *n_buckets, uint32_t *n_items,
                                   uint32_t *region_start, uint32_t *fill, uint32_t *work_page, uint32_t *work_slot,
                                   uint8_t *work_qcol, uint8_t *page_bin, uint8_t *page_narrow);
/* Alternative with a single collective: all-gather the exchange region (device pointer + length in
 * 8-byte words) of every rank into `gathered` (rank-major, n_ranks * words) and merge locally. */
tskv_status tskvgpu_scan_exchange_view(tskv_ctx *ctx, tskv_scan *scan, uint64_t *out_dptr, uint64_t *out_words);
tskv_status tskvgpu_scan_merge_gathered(tskv_ctx *ctx, tskv_scan *scan, uint64_t gathered_dptr, uint32_t n_ranks);

/* ---- multi-GPU inside the library: series sharded over ranks (one context = one GPU = one rank), NCCL for the one
 * exchange step. The reference shards series the same way (hash(SeriesKey) % n_shards, common/models/src/meta_data.rs:81-85)
 * and merges per-partition partial aggregates in DataFusion's final AggregateExec.
 *   tskvgpu_comm_unique_id  rank 0: ncclGetUniqueId; the host runtime hands the 128 bytes to the other ranks
 *   tskvgpu_comm_init       every rank: ncclCommInitRank on the context's device (collective: all ranks call it)
 *   tskvgpu_scan_exchange   after tskvgpu_scan_enqueue, every rank: ONE ncclAllGather of the scan's exchange region on
 *                           the context stream + the local merge (== exchange_view + merge_gathered). Queries of a
 *                           multi-rank scan carry TSKV_QUERY_MULTI_RANK and the global series_ids list.
 * libnccl.so.2 is loaded on first use (dlopen), so single-GPU users need no NCCL. */
#define TSKV_NCCL_UNIQUE_ID_BYTES 128
tskv_status tskvgpu_comm_unique_id(uint8_t out_id[TSKV_NCCL_UNIQUE_ID_BYTES]);
tskv_status tskvgpu_comm_init(tskv_ctx *ctx, const uint8_t id[TSKV_NCCL_UNIQUE_ID_BYTES], int32_t rank, int32_t n_ranks);
void tskvgpu_comm_destroy(tskv_ctx *ctx);
tskv_status tskvgpu_scan_exchange(tskv_ctx *ctx, tskv_scan *scan);
/* Snapshot the local first/last keys before they are all-reduced in place (multi-GPU only). */
tskv_status tskvgpu_scan_snapshot_keys(tskv_ctx *ctx, tskv_scan *scan);
/* Zero every first/last value whose local key (snapshot) lost the key all-reduce. */
tskv_status tskvgpu_scan_mask_values(tskv_ctx *ctx, tskv_scan *scan);
tskv_status tskvgpu_scan_finalize(tskv_ctx *ctx, tskv_scan *scan, uint64_t *out_values,
                                  uint8_t *out_validity);
/* Same as finalize but leaves the dense result on the device (no D2H): device pointers out. */
tskv_status tskvgpu_scan_finalize_device(tskv_ctx *ctx, tskv_scan *scan, uint64_t *out_values_dptr,
                                         uint64_t *out_validity_dptr);
void tskvgpu_scan_destroy(tskv_ctx *ctx, tskv_scan *scan);

/* ---- sliding windows: time_window(time, window, slide[, start_time]) --------------------------
 * The reference expands every row into k = ceil(window / slide) copies, one per window starting at
 * last_start(t) - i * slide (i < k), last_start(t) = t - ((t - start_time % window) + slide) % slide with truncating %
 * and wrapping arithmetic (build_sliding_window_plan, query_server/query/src/extension/analyse/transform_time_window.rs:
 * 251-393). These calls decode, filter and aggregate each row once, into panes one slide wide, and fold every run of k
 * consecutive panes into a window. The query's fields keep their meaning: width = window, origin = start_time; output
 * bucket j is the window starting at first_bucket_start + j * slide (n_buckets windows; tskvgpu_query_output_layout
 * describes the result). Every window of every selected row must lie on that grid, else TSKV_ERR_BUCKET_RANGE. The scan
 * returned works with every tskvgpu_scan_* call above. slide == width is the tumbling scan (tskvgpu_scan_prepare).
 * Refused before any launch:
 *   TSKV_ERR_INVALID_ARG   slide <= 0, width <= 0, k > 100 ("Too many overlapping windows"), n_buckets < k, or a grid
 *                          n_buckets * slide wider than 2^63
 *   TSKV_ERR_UNSUPPORTED   FIRST / LAST; slide > width; width >= 2^61; width % slide != 0 when a row the query can
 *                          select (time ranges x the page set's time bounds) has t - start_time % window + slide < 0, or
 *                          that dividend or t + window wraps (there the reference drops copies by the window-0 test:
 *                          see DESIGN.md section 7) */
tskv_status tskvgpu_scan_prepare_sliding(tskv_ctx *ctx, const tskv_pages *pages, const tskv_query *q,
                                         int64_t slide, tskv_scan **out_scan);
tskv_status tskvgpu_scan_aggregate_sliding(tskv_ctx *ctx, const tskv_pages *pages, const tskv_query *q,
                                           int64_t slide, uint64_t *out_values, uint8_t *out_validity);

/* ---- GROUP BY <tags>[, bucket] ---------------------------------------------------------------
 * Tags are not stored in pages: SeriesReader appends them per series from the SeriesKey (tskv/src/reader/series.rs:
 * 55-90,146-154), so grouping by a set of tags is a grouping of series the host knows before the scan.
 * group_ids[slot] in [0, n_groups) is the group of the slot-th selected series (q->series_ids order; every series of the
 * page set in ascending id order when series_ids == NULL). Output cell c = group * n_buckets + bucket. A group's cell
 * aggregates every selected row of every series in the group that falls in the bucket / window; FIRST / LAST pick the
 * group's earliest / latest row, ties to the lower slot (the keys and budget of the ungrouped scan), so group g's result
 * equals the ungrouped scan whose series_ids are g's members. A group without a selected row reads like an empty bucket.
 * slide == 0 or slide == q->width: tumbling buckets; otherwise the sliding windows (and every refusal) of
 * tskvgpu_scan_prepare_sliding. The scan returned works with every tskvgpu_scan_* call above; multi-rank scans
 * (TSKV_QUERY_MULTI_RANK) pass the same global series_ids and the same group_ids on every rank.
 * Refused before any launch with TSKV_ERR_INVALID_ARG: group_ids == NULL, n_groups == 0, a group id >= n_groups,
 * q->group_by_series != 0, or n_groups * n_buckets > TSKV_MAX_GROUPED_CELLS. */
#define TSKV_MAX_GROUPED_CELLS 0xffffffffu
tskv_status tskvgpu_query_output_layout_grouped(const tskv_pages *pages, const tskv_query *q,
                                                const uint32_t *group_ids, uint32_t n_groups, tskv_output_layout *out);
tskv_status tskvgpu_scan_prepare_grouped(tskv_ctx *ctx, const tskv_pages *pages, const tskv_query *q,
                                         const uint32_t *group_ids, uint32_t n_groups, int64_t slide, tskv_scan **out);
tskv_status tskvgpu_scan_aggregate_grouped(tskv_ctx *ctx, const tskv_pages *pages, const tskv_query *q,
                                           const uint32_t *group_ids, uint32_t n_groups, int64_t slide,
                                           uint64_t *out_values, uint8_t *out_validity);

/* ---- explicit time-bucket edges: GROUP BY date_trunc(unit, time) and other irregular grids ----------------
 * Time bucket b (0 <= b < q->n_buckets) is the half-open interval [edges[b], edges[b + 1]). edges holds q->n_buckets + 1
 * strictly increasing timestamps (the time column's unit). q->width, q->origin and q->first_bucket_start must be 0: the
 * edges replace them. A selected row outside [edges[0], edges[n_buckets]) is TSKV_ERR_BUCKET_RANGE, as a row off the
 * tumbling grid is. group_ids == NULL: no tag groups (group_by_series may be set). Otherwise group_ids / n_groups work as in
 * tskvgpu_scan_prepare_grouped. FIRST / LAST: (page, time bucket) runs and tie-break keys as in the tumbling scan, with
 * rel = t - edges[b] + 1 and the 62-bit budget taken from the longest bucket. The scan returned works with every tskvgpu_scan_*
 * call, including TSKV_QUERY_MULTI_RANK exchange (every rank passes the same edges).
 * Refused before any launch:
 *   TSKV_ERR_INVALID_ARG   edges == NULL, n_buckets == 0, edges not strictly increasing, edges[n] - edges[0] >= 2^63,
 *                          width / origin / first_bucket_start != 0, a bad group map, or n_groups * n_buckets > TSKV_MAX_GROUPED_CELLS
 *   TSKV_ERR_UNSUPPORTED   FIRST / LAST across series whose keys do not fit (bits(longest bucket) + slot bits > 62) */
tskv_status tskvgpu_query_output_layout_edges(const tskv_pages *pages, const tskv_query *q, const int64_t *edges,
                                              const uint32_t *group_ids, uint32_t n_groups, tskv_output_layout *out);
tskv_status tskvgpu_scan_prepare_edges(tskv_ctx *ctx, const tskv_pages *pages, const tskv_query *q, const int64_t *edges,
                                       const uint32_t *group_ids, uint32_t n_groups, tskv_scan **out_scan);
tskv_status tskvgpu_scan_aggregate_edges(tskv_ctx *ctx, const tskv_pages *pages, const tskv_query *q, const int64_t *edges,
                                         const uint32_t *group_ids, uint32_t n_groups, uint64_t *out_values, uint8_t *out_validity);

/* ---- labelled time buckets: GROUP BY date_part(unit, time) / EXTRACT(unit FROM time) ---------------------------------
 * n_edge + 1 strictly increasing edges cut time into edge buckets [edges[b], edges[b + 1]), exactly as in
 * tskvgpu_scan_prepare_edges, and labels[b] < q->n_buckets names the output bucket of edge bucket b: q->n_buckets is the
 * number of output buckets per group. A selected row in edge bucket b aggregates into cell group * q->n_buckets + labels[b].
 * Several edge buckets may share a label (the hour of the day over many days); an output bucket that no edge bucket maps
 * to reads like an empty bucket. A selected row outside [edges[0], edges[n_edge]) is TSKV_ERR_BUCKET_RANGE. COUNT, SUM,
 * MIN, MAX and MEAN are those of every other scan; labels[b] = b with q->n_buckets = n_edge gives the edge scan's result.
 * group_ids / n_groups and group_by_series as in tskvgpu_scan_prepare_edges. The scan returned works with every
 * tskvgpu_scan_* call, including TSKV_QUERY_MULTI_RANK exchange (every rank passes the same edges and labels).
 * Refused before any launch:
 *   TSKV_ERR_INVALID_ARG   labels == NULL, a label >= q->n_buckets, q->n_buckets == 0, and every refusal of the edges
 *                          calls (with n_edge for their n_buckets; n_groups * q->n_buckets > TSKV_MAX_GROUPED_CELLS)
 *   TSKV_ERR_UNSUPPORTED   FIRST / LAST (the reference takes each record batch's earliest row per label, so the NULL rule at
 *                          that row acts across the page's edge buckets of one label: DESIGN.md section 7) */
tskv_status tskvgpu_query_output_layout_labels(const tskv_pages *pages, const tskv_query *q, const int64_t *edges,
                                               uint32_t n_edge, const uint32_t *labels, const uint32_t *group_ids,
                                               uint32_t n_groups, tskv_output_layout *out);
tskv_status tskvgpu_scan_prepare_labels(tskv_ctx *ctx, const tskv_pages *pages, const tskv_query *q, const int64_t *edges,
                                        uint32_t n_edge, const uint32_t *labels, const uint32_t *group_ids, uint32_t n_groups,
                                        tskv_scan **out_scan);
tskv_status tskvgpu_scan_aggregate_labels(tskv_ctx *ctx, const tskv_pages *pages, const tskv_query *q, const int64_t *edges,
                                          uint32_t n_edge, const uint32_t *labels, const uint32_t *group_ids, uint32_t n_groups,
                                          uint64_t *out_values, uint8_t *out_validity);

/* Library version / build info ("tskv-b200 <semver> sm_90a"). */
const char *tskvgpu_version(void);

#ifdef __cplusplus
} /* extern "C" */
#endif
#endif /* TSKV_GPU_H_ */
