//! Raw bindings of `include/tskv_gpu.h` (keep in sync: tests/test_cabi_symbols.py compares the two).
#![allow(non_camel_case_types)]
use std::os::raw::c_char;

pub type tskv_status = i32;
pub const TSKV_OK: tskv_status = 0;
pub const TSKV_ERR_INVALID_ARG: tskv_status = 1;
pub const TSKV_ERR_BAD_ENCODING: tskv_status = 2;
pub const TSKV_ERR_SHORT_BLOCK: tskv_status = 3;
pub const TSKV_ERR_CRC_MISMATCH: tskv_status = 4;
pub const TSKV_ERR_BITSET_MISMATCH: tskv_status = 5;
pub const TSKV_ERR_UNSUPPORTED: tskv_status = 6;
pub const TSKV_ERR_BUCKET_RANGE: tskv_status = 7;
pub const TSKV_ERR_CUDA: tskv_status = 8;
pub const TSKV_ERR_NCCL: tskv_status = 9;
pub const TSKV_ERR_OOM: tskv_status = 10;
pub const TSKV_ERR_BAD_LENGTH: tskv_status = 11;
pub const TSKV_ERR_PAGE_FORMAT: tskv_status = 12;

pub const TSKV_PT_TIME: u8 = 0;
pub const TSKV_PT_I64: u8 = 1;
pub const TSKV_PT_U64: u8 = 2;
pub const TSKV_PT_F64: u8 = 3;
pub const TSKV_PT_BOOL: u8 = 4;

pub const TSKV_AGG_COUNT: u8 = 1 << 0;
pub const TSKV_AGG_SUM: u8 = 1 << 1;
pub const TSKV_AGG_MIN: u8 = 1 << 2;
pub const TSKV_AGG_MAX: u8 = 1 << 3;
pub const TSKV_AGG_MEAN: u8 = 1 << 4;
pub const TSKV_AGG_FIRST: u8 = 1 << 5;
pub const TSKV_AGG_LAST: u8 = 1 << 6;
/// f64 sum of squared deviations from the cell mean (the variance state; two passes, see tskv_gpu.h).
pub const TSKV_AGG_M2: u8 = 1 << 7;
/// At most this many column pairs (tskv_query.n_pairs; covariance / correlation, see tskv_gpu.h).
pub const TSKV_MAX_PAIRS: u32 = 8;
/// At most this many medians; their count sits in bits 8..15 of tskv_query.reserved (see tskv_gpu.h).
pub const TSKV_MAX_MEDIANS: u32 = 8;
/// A scan with medians holds at most this many cells times medians (1 KiB of histogram each).
pub const TSKV_MAX_MEDIAN_CELLS: u64 = 1 << 22;
/// TSKV_QUERY_MEDIANS(n): the flags-word bits of n medians.
pub const fn tskv_query_medians(n: u32) -> u32 {
    (n & 0xff) << 8
}
/// TSKV_QUERY_N_MEDIANS(flags): the medians of a flags word.
pub const fn tskv_query_n_medians(flags: u32) -> u32 {
    (flags >> 8) & 0xff
}
/// At most this many increases; their count sits in bits 16..23 of tskv_query.reserved (see tskv_gpu.h).
pub const TSKV_MAX_INCREASES: u32 = 8;
/// TSKV_QUERY_INCREASES(n): the flags-word bits of n increases.
pub const fn tskv_query_increases(n: u32) -> u32 {
    (n & 0xff) << 16
}
/// TSKV_QUERY_N_INCREASES(flags): the increases of a flags word.
pub const fn tskv_query_n_increases(flags: u32) -> u32 {
    (flags >> 16) & 0xff
}
/// At most this many modes; their count sits in bits 24..27 of tskv_query.reserved (see tskv_gpu.h).
pub const TSKV_MAX_MODES: u32 = 8;
/// At most this many distinct counts; their count sits in bits 28..31 of tskv_query.reserved.
pub const TSKV_MAX_DISTINCTS: u32 = 8;
/// Modes and distincts are refused when their operands' selectable rows could reach this many.
pub const TSKV_MAX_SORTED_ROWS: u32 = 0x7fff_ffff;
/// TSKV_QUERY_MODES(n): the flags-word bits of n modes.
pub const fn tskv_query_modes(n: u32) -> u32 {
    (n & 0xf) << 24
}
/// TSKV_QUERY_N_MODES(flags): the modes of a flags word.
pub const fn tskv_query_n_modes(flags: u32) -> u32 {
    (flags >> 24) & 0xf
}
/// TSKV_QUERY_DISTINCTS(n): the flags-word bits of n distinct counts.
pub const fn tskv_query_distincts(n: u32) -> u32 {
    (n & 0xf) << 28
}
/// TSKV_QUERY_N_DISTINCTS(flags): the distinct counts of a flags word.
pub const fn tskv_query_n_distincts(flags: u32) -> u32 {
    (flags >> 28) & 0xf
}
/// At most this many gauges (gauge_agg(time, x)); their count sits in bits 1..4 of tskv_query.reserved. Their operands
/// follow the distincts' operands in `columns`; each adds 9 outputs: n, then (t, v) of the first, second, penultimate
/// and last point.
pub const TSKV_MAX_GAUGES: u32 = 8;
/// TSKV_QUERY_GAUGES(n): the flags-word bits of n gauges.
pub const fn tskv_query_gauges(n: u32) -> u32 {
    (n & 0xf) << 1
}
/// TSKV_QUERY_N_GAUGES(flags): the gauges of a flags word.
pub const fn tskv_query_n_gauges(flags: u32) -> u32 {
    (flags >> 1) & 0xf
}
/// At most this many state aggs (compact_state_agg(time, x)); their count sits in bits 5..7 of tskv_query.reserved (with
/// them the flags word is full). Their operands follow the gauges' operands in `columns`; each adds 1 output (the cell's
/// map entries), and tskvgpu_scan_state_durations returns the maps.
pub const TSKV_MAX_STATE_AGGS: u32 = 7;
/// TSKV_QUERY_STATE_AGGS(n): the flags-word bits of n state aggs.
pub const fn tskv_query_state_aggs(n: u32) -> u32 {
    (n & 0x7) << 5
}
/// TSKV_QUERY_N_STATE_AGGS(flags): the state aggs of a flags word.
pub const fn tskv_query_n_state_aggs(flags: u32) -> u32 {
    (flags >> 5) & 0x7
}
/// A state agg operand's agg_mask (instead of 0): the agg computes state_agg(time, x)'s periods as well as its map, and
/// tskvgpu_scan_state_periods returns them.
pub const TSKV_STATE_PERIODS: u32 = 1 << 7;

pub const TSKV_UPLOAD_VERIFY_CRC: u32 = 1;
pub const TSKV_UPLOAD_HOST_RESIDENT: u32 = 2;
pub const TSKV_UPLOAD_VERIFY_ON_READ: u32 = 4;
pub const TSKV_TOMB_ALL: u32 = 0xffff_ffff;
pub const TSKV_QUERY_MULTI_RANK: u32 = 1;
pub const TSKV_MAX_GROUPED_CELLS: u64 = 0xffff_ffff;
pub const TSKV_MAX_PREDICATES: usize = 8;
pub const TSKV_NCCL_UNIQUE_ID_BYTES: usize = 128;

pub const TSKV_CMP_EQ: u8 = 0;
pub const TSKV_CMP_NE: u8 = 1;
pub const TSKV_CMP_LT: u8 = 2;
pub const TSKV_CMP_LE: u8 = 3;
pub const TSKV_CMP_GT: u8 = 4;
pub const TSKV_CMP_GE: u8 = 5;

#[repr(C)]
pub struct tskv_ctx {
    _private: [u8; 0],
}
#[repr(C)]
pub struct tskv_pages {
    _private: [u8; 0],
}
#[repr(C)]
pub struct tskv_scan {
    _private: [u8; 0],
}

/// `PageWriteSpec{offset,size,meta}` + the bytes it addresses (tskv/src/tsm/page.rs:599-620). 24 bytes.
#[repr(C)]
#[derive(Clone, Copy, Debug, Default)]
pub struct tskv_page_desc {
    pub offset: u64,
    pub size: u32,
    pub num_values: u32,
    pub series_id: u32,
    pub column_id: u16,
    pub phys_type: u8,
    pub reserved: u8,
}

/// Closed interval, `TimeRange{min_ts,max_ts}` (common/models/src/predicate/domain.rs:35-98).
#[repr(C)]
#[derive(Clone, Copy, Debug, Default, PartialEq, Eq)]
pub struct tskv_time_range {
    pub min_ts: i64,
    pub max_ts: i64,
}

#[repr(C)]
#[derive(Clone, Copy, Debug, Default)]
pub struct tskv_agg_column {
    pub column_id: u16,
    pub phys_type: u8,
    pub agg_mask: u8,
}

#[repr(C)]
#[derive(Clone, Copy, Debug, Default)]
pub struct tskv_field_predicate {
    pub column_id: u16,
    pub phys_type: u8,
    pub op: u8,
    pub reserved: u32,
    pub value: u64,
}

#[repr(C)]
#[derive(Clone, Copy, Debug)]
pub struct tskv_tombstone {
    pub series_id: u32,
    pub column_id: u32,
    pub min_ts: i64,
    pub max_ts: i64,
}

pub const TSKV_STATS_MINMAX: u32 = 1;
/// `PageMeta.statistics` of one page (tskv/src/tsm/page.rs:599-613): bit patterns of the page's physical type.
#[repr(C)]
#[derive(Clone, Copy, Debug, Default)]
pub struct tskv_value_stats {
    pub min: u64,
    pub max: u64,
    pub flags: u32,
    pub reserved: u32,
}

#[repr(C)]
pub struct tskv_query {
    pub series_ids: *const u32,
    pub n_series: u32,
    pub n_time_ranges: u32,
    pub time_ranges: *const tskv_time_range,
    pub origin: i64,
    pub width: i64,
    pub first_bucket_start: i64,
    pub n_buckets: u32,
    pub group_by_series: u32,
    pub columns: *const tskv_agg_column,
    pub n_columns: u32,
    pub reserved: u32,
    pub predicates: *const tskv_field_predicate,
    pub n_predicates: u32,
    /// column pairs (covariance / correlation), operands after the projected columns; 0: none
    pub n_pairs: u32,
}

#[repr(C)]
#[derive(Clone, Copy, Debug, Default)]
pub struct tskv_output_layout {
    pub n_out: u64,
    pub n_groups: u64,
    pub n_cells: u64,
    pub bitmap_stride: u64,
    pub values_bytes: u64,
    pub validity_bytes: u64,
}

#[repr(C)]
#[derive(Clone, Copy, Debug, Default)]
pub struct tskv_counters {
    pub page_read_count: u64,
    pub page_read_bytes: u64,
    pub points_decoded: u64,
    pub rows_in_range: u64,
    pub elapsed_scan_ms: f64,
    pub elapsed_h2d_ms: f64,
    pub kernel_launches: u64,
    pub elapsed_fused_ms: f64,
    pub dominant_kernel_ms: f64,
    pub dominant_kernel_bytes: u64,
    pub dominant_kernel_bin: u64,
    pub h2d_bytes: u64,
    pub pruned_page_count: u64,
}

#[repr(C)]
#[derive(Clone, Copy, Debug, Default)]
pub struct tskv_partials_view {
    pub sum_i64_ptr: u64,
    pub sum_i64_len: u64,
    pub sum_f64_ptr: u64,
    pub sum_f64_len: u64,
    pub min_i64_ptr: u64,
    pub min_i64_len: u64,
    pub max_i64_ptr: u64,
    pub max_i64_len: u64,
    pub sel_val_ptr: u64,
    pub sel_val_len: u64,
    pub sel_first_len: u64,
    pub sel_last_len: u64,
}

// sizes the C header fixes (checked against ctypes in tests/test_cabi_symbols.py)
const _: () = assert!(std::mem::size_of::<tskv_page_desc>() == 24);
const _: () = assert!(std::mem::size_of::<tskv_time_range>() == 16);
const _: () = assert!(std::mem::size_of::<tskv_agg_column>() == 4);
const _: () = assert!(std::mem::size_of::<tskv_field_predicate>() == 16);
const _: () = assert!(std::mem::size_of::<tskv_tombstone>() == 24);
const _: () = assert!(std::mem::size_of::<tskv_value_stats>() == 24);
const _: () = assert!(std::mem::size_of::<tskv_query>() == 88);
const _: () = assert!(std::mem::size_of::<tskv_output_layout>() == 48);
const _: () = assert!(std::mem::size_of::<tskv_counters>() == 104);
const _: () = assert!(std::mem::size_of::<tskv_partials_view>() == 96);

extern "C" {
    pub fn tskvgpu_version() -> *const c_char;
    pub fn tskvgpu_ctx_create(device_id: i32, out_ctx: *mut *mut tskv_ctx) -> tskv_status;
    pub fn tskvgpu_ctx_destroy(ctx: *mut tskv_ctx);
    pub fn tskvgpu_last_error(ctx: *const tskv_ctx) -> *const c_char;
    pub fn tskvgpu_last_error_page(ctx: *const tskv_ctx) -> i64;
    pub fn tskvgpu_get_counters(ctx: *const tskv_ctx, out: *mut tskv_counters) -> tskv_status;
    pub fn tskvgpu_ctx_stream(ctx: *const tskv_ctx) -> u64;

    pub fn tskvgpu_upload_pages(
        ctx: *mut tskv_ctx,
        arena: *const u8,
        arena_len: u64,
        descs: *const tskv_page_desc,
        n_descs: u64,
        flags: u32,
        out_pages: *mut *mut tskv_pages,
    ) -> tskv_status;
    pub fn tskvgpu_pages_destroy(ctx: *mut tskv_ctx, pages: *mut tskv_pages);
    pub fn tskvgpu_pages_series_count(pages: *const tskv_pages) -> u64;
    pub fn tskvgpu_pages_set_time_bounds(
        ctx: *mut tskv_ctx,
        pages: *mut tskv_pages,
        bounds: *const tskv_time_range,
        n: u64,
    ) -> tskv_status;
    pub fn tskvgpu_pages_set_tombstones(
        ctx: *mut tskv_ctx,
        pages: *mut tskv_pages,
        tombs: *const tskv_tombstone,
        n_tombs: u64,
    ) -> tskv_status;
    /// `PageMeta.statistics` per descriptor: scans with field predicates prune by them (reader/chunk.rs:12-50).
    pub fn tskvgpu_pages_set_value_stats(
        ctx: *mut tskv_ctx,
        pages: *mut tskv_pages,
        stats: *const tskv_value_stats,
        n_descs: u64,
    ) -> tskv_status;
    /// File id of every column group: overlapping chunks of a series are merged (DataMerger, reader/merge.rs).
    pub fn tskvgpu_pages_set_chunk_files(
        ctx: *mut tskv_ctx,
        pages: *mut tskv_pages,
        cg_file_id: *const u64,
        n_cg: u64,
    ) -> tskv_status;

    pub fn tskvgpu_decode_pages(
        ctx: *mut tskv_ctx,
        pages: *const tskv_pages,
        first_page: u64,
        n_pages: u64,
        out_values: *mut u64,
        out_validity: *mut u8,
    ) -> tskv_status;

    pub fn tskvgpu_query_output_layout(
        pages: *const tskv_pages,
        q: *const tskv_query,
        out: *mut tskv_output_layout,
    ) -> tskv_status;
    pub fn tskvgpu_scan_aggregate(
        ctx: *mut tskv_ctx,
        pages: *const tskv_pages,
        q: *const tskv_query,
        out_values: *mut u64,
        out_validity: *mut u8,
    ) -> tskv_status;

    pub fn tskvgpu_scan_prepare(
        ctx: *mut tskv_ctx,
        pages: *const tskv_pages,
        q: *const tskv_query,
        out_scan: *mut *mut tskv_scan,
    ) -> tskv_status;
    pub fn tskvgpu_scan_prepare_sliding(
        ctx: *mut tskv_ctx,
        pages: *const tskv_pages,
        q: *const tskv_query,
        slide: i64,
        out_scan: *mut *mut tskv_scan,
    ) -> tskv_status;
    pub fn tskvgpu_scan_aggregate_sliding(
        ctx: *mut tskv_ctx,
        pages: *const tskv_pages,
        q: *const tskv_query,
        slide: i64,
        out_values: *mut u64,
        out_validity: *mut u8,
    ) -> tskv_status;
    pub fn tskvgpu_query_output_layout_grouped(
        pages: *const tskv_pages,
        q: *const tskv_query,
        group_ids: *const u32,
        n_groups: u32,
        out: *mut tskv_output_layout,
    ) -> tskv_status;
    pub fn tskvgpu_scan_prepare_grouped(
        ctx: *mut tskv_ctx,
        pages: *const tskv_pages,
        q: *const tskv_query,
        group_ids: *const u32,
        n_groups: u32,
        slide: i64,
        out_scan: *mut *mut tskv_scan,
    ) -> tskv_status;
    pub fn tskvgpu_scan_aggregate_grouped(
        ctx: *mut tskv_ctx,
        pages: *const tskv_pages,
        q: *const tskv_query,
        group_ids: *const u32,
        n_groups: u32,
        slide: i64,
        out_values: *mut u64,
        out_validity: *mut u8,
    ) -> tskv_status;
    pub fn tskvgpu_query_output_layout_edges(
        pages: *const tskv_pages,
        q: *const tskv_query,
        edges: *const i64,
        group_ids: *const u32,
        n_groups: u32,
        out: *mut tskv_output_layout,
    ) -> tskv_status;
    pub fn tskvgpu_scan_prepare_edges(
        ctx: *mut tskv_ctx,
        pages: *const tskv_pages,
        q: *const tskv_query,
        edges: *const i64,
        group_ids: *const u32,
        n_groups: u32,
        out_scan: *mut *mut tskv_scan,
    ) -> tskv_status;
    pub fn tskvgpu_scan_aggregate_edges(
        ctx: *mut tskv_ctx,
        pages: *const tskv_pages,
        q: *const tskv_query,
        edges: *const i64,
        group_ids: *const u32,
        n_groups: u32,
        out_values: *mut u64,
        out_validity: *mut u8,
    ) -> tskv_status;
    pub fn tskvgpu_query_output_layout_labels(
        pages: *const tskv_pages,
        q: *const tskv_query,
        edges: *const i64,
        n_edge: u32,
        labels: *const u32,
        group_ids: *const u32,
        n_groups: u32,
        out: *mut tskv_output_layout,
    ) -> tskv_status;
    pub fn tskvgpu_scan_prepare_labels(
        ctx: *mut tskv_ctx,
        pages: *const tskv_pages,
        q: *const tskv_query,
        edges: *const i64,
        n_edge: u32,
        labels: *const u32,
        group_ids: *const u32,
        n_groups: u32,
        out_scan: *mut *mut tskv_scan,
    ) -> tskv_status;
    pub fn tskvgpu_scan_aggregate_labels(
        ctx: *mut tskv_ctx,
        pages: *const tskv_pages,
        q: *const tskv_query,
        edges: *const i64,
        n_edge: u32,
        labels: *const u32,
        group_ids: *const u32,
        n_groups: u32,
        out_values: *mut u64,
        out_validity: *mut u8,
    ) -> tskv_status;
    pub fn tskvgpu_scan_run(ctx: *mut tskv_ctx, scan: *mut tskv_scan) -> tskv_status;
    pub fn tskvgpu_scan_enqueue(ctx: *mut tskv_ctx, scan: *mut tskv_scan) -> tskv_status;
    pub fn tskvgpu_scan_sync(ctx: *mut tskv_ctx, scan: *mut tskv_scan) -> tskv_status;
    pub fn tskvgpu_scan_partials(ctx: *mut tskv_ctx, scan: *mut tskv_scan, out: *mut tskv_partials_view) -> tskv_status;
    pub fn tskvgpu_scan_work_list(
        ctx: *mut tskv_ctx,
        scan: *mut tskv_scan,
        n_buckets: *mut u32,
        n_items: *mut u32,
        region_start: *mut u32,
        fill: *mut u32,
        work_page: *mut u32,
        work_slot: *mut u32,
        work_qcol: *mut u8,
        page_bin: *mut u8,
        page_narrow: *mut u8,
    ) -> tskv_status;
    pub fn tskvgpu_scan_state_durations(
        ctx: *mut tskv_ctx,
        scan: *mut tskv_scan,
        k: u32,
        offsets: *mut u64,
        states: *mut u64,
        state_valid: *mut u8,
        durations: *mut i64,
        n_entries: *mut u64,
    ) -> tskv_status;
    pub fn tskvgpu_scan_state_periods(
        ctx: *mut tskv_ctx,
        scan: *mut tskv_scan,
        k: u32,
        offsets: *mut u64,
        states: *mut u64,
        state_valid: *mut u8,
        starts: *mut i64,
        ends: *mut i64,
        n_periods: *mut u64,
    ) -> tskv_status;
    pub fn tskvgpu_scan_exchange_view(
        ctx: *mut tskv_ctx,
        scan: *mut tskv_scan,
        out_dptr: *mut u64,
        out_words: *mut u64,
    ) -> tskv_status;
    pub fn tskvgpu_scan_merge_gathered(
        ctx: *mut tskv_ctx,
        scan: *mut tskv_scan,
        gathered_dptr: u64,
        n_ranks: u32,
    ) -> tskv_status;
    pub fn tskvgpu_scan_snapshot_keys(ctx: *mut tskv_ctx, scan: *mut tskv_scan) -> tskv_status;
    pub fn tskvgpu_scan_mask_values(ctx: *mut tskv_ctx, scan: *mut tskv_scan) -> tskv_status;
    pub fn tskvgpu_scan_finalize(
        ctx: *mut tskv_ctx,
        scan: *mut tskv_scan,
        out_values: *mut u64,
        out_validity: *mut u8,
    ) -> tskv_status;
    pub fn tskvgpu_scan_finalize_device(
        ctx: *mut tskv_ctx,
        scan: *mut tskv_scan,
        out_values_dptr: *mut u64,
        out_validity_dptr: *mut u64,
    ) -> tskv_status;
    pub fn tskvgpu_scan_destroy(ctx: *mut tskv_ctx, scan: *mut tskv_scan);

    pub fn tskvgpu_comm_unique_id(out_id: *mut u8) -> tskv_status;
    pub fn tskvgpu_comm_init(ctx: *mut tskv_ctx, id: *const u8, rank: i32, n_ranks: i32) -> tskv_status;
    pub fn tskvgpu_comm_destroy(ctx: *mut tskv_ctx);
    pub fn tskvgpu_scan_exchange(ctx: *mut tskv_ctx, scan: *mut tskv_scan) -> tskv_status;
}
