//! Safe wrapper over `libtskv_gpu.so`, the H100-native replacement of ONE path of cnosdb's `tskv` crate:
//! TSM page decode -> time-range / series / field-predicate filter -> time-bucketed aggregate.
//!
//! The reference has no FFI; the seam is the `BatchReader` tree built by
//! `SeriesGroupBatchReaderFactory::create` (tskv/src/reader/iterator.rs:123-264) and polled through
//! `BatchReader::process` (tskv/src/reader/mod.rs:159-164). A `GpuAggregateBatchReader` inside the `tskv` crate
//! (INTEGRATION.md section 3 shows it) implements that trait with the types below:
//!
//! ```text
//! GpuEngine::new(device)                       one per GPU, shared by all tokio workers (thread-safe)
//!   .upload_pages(arena, descs, flags)         TsmReader::read_adjacent_pages + Page::crc_validation
//!   PageSet::set_time_bounds / set_tombstones  ColumnGroup::time_range(), TsmTombstone cache
//!   .scan_aggregate(&pages, &Query)            decode_pages + DataFilter + AggregateExec, one call
//! ```
//!
//! Blocking calls: wrap them in `tokio::task::spawn_blocking` like every other file read of the reader tree.
//! This crate is source only in the repository's image (no Rust toolchain there); the same call sequence is compiled
//! and tested through the C++ mirror (`cnosdb_b200/csrc/host/batch_reader.{h,cc}`) and the ctypes binding.
pub mod sys;

use std::ffi::CStr;
use std::fmt;
use std::marker::PhantomData;
use std::sync::Arc;

pub use sys::{tskv_agg_column, tskv_field_predicate, tskv_page_desc, tskv_time_range, tskv_tombstone};
pub use sys::{tskv_query_medians, tskv_query_n_medians, TSKV_MAX_MEDIANS, TSKV_MAX_MEDIAN_CELLS};
pub use sys::{tskv_query_increases, tskv_query_n_increases, TSKV_MAX_INCREASES};
pub use sys::{tskv_query_distincts, tskv_query_modes, tskv_query_n_distincts, tskv_query_n_modes};
pub use sys::{TSKV_MAX_DISTINCTS, TSKV_MAX_MODES, TSKV_MAX_SORTED_ROWS};
pub use sys::{tskv_query_gauges, tskv_query_n_gauges, TSKV_MAX_GAUGES};
pub use sys::{tskv_query_n_state_aggs, tskv_query_state_aggs, TSKV_MAX_STATE_AGGS, TSKV_STATE_PERIODS};

/// What a failed call reports; maps onto `TskvError` as INTEGRATION.md section 2 lists.
#[derive(Debug, Clone)]
pub struct GpuError {
    pub status: sys::tskv_status,
    pub message: String,
    /// descriptor index of the page a decode / CRC error was found in, or -1
    pub page: i64,
}

impl GpuError {
    /// `TskvError::Decode` class (codec error strings of timestamp.rs / integer.rs / float.rs)
    pub fn is_decode(&self) -> bool {
        matches!(
            self.status,
            sys::TSKV_ERR_BAD_ENCODING
                | sys::TSKV_ERR_SHORT_BLOCK
                | sys::TSKV_ERR_BITSET_MISMATCH
                | sys::TSKV_ERR_UNSUPPORTED
                | sys::TSKV_ERR_BAD_LENGTH
                | sys::TSKV_ERR_PAGE_FORMAT
        )
    }
    /// `TskvError::TsmPageFileHashCheckFailed` (tskv/src/tsm/page.rs:66-73)
    pub fn is_crc(&self) -> bool {
        self.status == sys::TSKV_ERR_CRC_MISMATCH
    }
}

impl fmt::Display for GpuError {
    fn fmt(&self, f: &mut fmt::Formatter<'_>) -> fmt::Result {
        write!(f, "tskv-gpu status {} (page {}): {}", self.status, self.page, self.message)
    }
}
impl std::error::Error for GpuError {}

pub type GpuResult<T> = Result<T, GpuError>;

/// One CUDA device + stream (`tskv_ctx`). Calls on one engine are serialised inside the library.
pub struct GpuEngine {
    ctx: *mut sys::tskv_ctx,
}
// SAFETY: the library guards every entry point of a context with its own mutex and never relies on a thread-local
// current device (include/tskv_gpu.h, "Conventions").
unsafe impl Send for GpuEngine {}
unsafe impl Sync for GpuEngine {}

impl GpuEngine {
    pub fn new(device: i32) -> GpuResult<Arc<Self>> {
        let mut ctx = std::ptr::null_mut();
        let st = unsafe { sys::tskvgpu_ctx_create(device, &mut ctx) };
        if st != sys::TSKV_OK {
            return Err(GpuError { status: st, message: format!("no usable CUDA device {device}"), page: -1 });
        }
        Ok(Arc::new(Self { ctx }))
    }

    fn check(&self, st: sys::tskv_status) -> GpuResult<()> {
        if st == sys::TSKV_OK {
            return Ok(());
        }
        let message = unsafe { CStr::from_ptr(sys::tskvgpu_last_error(self.ctx)) }.to_string_lossy().into_owned();
        let page = unsafe { sys::tskvgpu_last_error_page(self.ctx) };
        Err(GpuError { status: st, message, page })
    }

    pub fn counters(&self) -> sys::tskv_counters {
        let mut c = sys::tskv_counters::default();
        unsafe { sys::tskvgpu_get_counters(self.ctx, &mut c) };
        c
    }

    /// `TsmReader::read_adjacent_pages` + `Page::crc_validation`: `arena` holds the raw page bytes, `descs` lists them
    /// column group by column group (TIME page first). With `TSKV_UPLOAD_HOST_RESIDENT` the bytes stay where they are
    /// (page-locked by the library) and must outlive the returned page set - hence the lifetime.
    pub fn upload_pages<'a>(self: &Arc<Self>, arena: &'a [u8], descs: &[tskv_page_desc], flags: u32) -> GpuResult<PageSet<'a>> {
        let mut pages = std::ptr::null_mut();
        let st = unsafe {
            sys::tskvgpu_upload_pages(self.ctx, arena.as_ptr(), arena.len() as u64, descs.as_ptr(), descs.len() as u64, flags, &mut pages)
        };
        self.check(st)?;
        Ok(PageSet { engine: self.clone(), pages, _arena: PhantomData })
    }

    /// The end-to-end call a `BatchReader::process()` makes: query arguments H2D, fused scan, dense result D2H.
    pub fn scan_aggregate(&self, pages: &PageSet<'_>, q: &Query) -> GpuResult<AggregateResult> {
        let raw = q.as_raw()?;
        let layout = self.output_layout(pages, q, &raw)?;
        let mut values = vec![0u64; (layout.n_out * layout.n_cells) as usize];
        let mut validity = vec![0u8; layout.validity_bytes as usize];
        self.check(unsafe {
            match (&q.groups, q.slide) {
                (Some((ids, n)), slide) => sys::tskvgpu_scan_aggregate_grouped(
                    self.ctx, pages.pages, &raw, ids.as_ptr(), *n, slide.unwrap_or(0), values.as_mut_ptr(), validity.as_mut_ptr()),
                (None, None) => sys::tskvgpu_scan_aggregate(self.ctx, pages.pages, &raw, values.as_mut_ptr(), validity.as_mut_ptr()),
                (None, Some(slide)) => {
                    sys::tskvgpu_scan_aggregate_sliding(self.ctx, pages.pages, &raw, slide, values.as_mut_ptr(), validity.as_mut_ptr())
                }
            }
        })?;
        Ok(AggregateResult { layout, values, validity })
    }

    /// `scan_aggregate` for a query with state aggs (`Query::n_state_aggs`): the dense result (each state agg's output is
    /// the cell's number of map entries), every state agg's maps, which the one-shot call does not return, and the
    /// periods of every state agg whose operand has agg_mask TSKV_STATE_PERIODS (None for the others).
    pub fn scan_aggregate_states(
        &self,
        pages: &PageSet<'_>,
        q: &Query,
    ) -> GpuResult<(AggregateResult, Vec<StateDurations>, Vec<Option<StatePeriods>>)> {
        let raw = q.as_raw()?;
        let layout = self.output_layout(pages, q, &raw)?;
        let mut scan = std::ptr::null_mut();
        self.check(unsafe {
            match (&q.groups, q.slide) {
                (Some((ids, n)), slide) => {
                    sys::tskvgpu_scan_prepare_grouped(self.ctx, pages.pages, &raw, ids.as_ptr(), *n, slide.unwrap_or(0), &mut scan)
                }
                (None, None) => sys::tskvgpu_scan_prepare(self.ctx, pages.pages, &raw, &mut scan),
                (None, Some(slide)) => sys::tskvgpu_scan_prepare_sliding(self.ctx, pages.pages, &raw, slide, &mut scan),
            }
        })?;
        let mut values = vec![0u64; (layout.n_out * layout.n_cells) as usize];
        let mut validity = vec![0u8; layout.validity_bytes as usize];
        let mut maps = Vec::with_capacity(q.n_state_aggs as usize);
        let mut periods = Vec::with_capacity(q.n_state_aggs as usize);
        let ops = &q.columns[q.columns.len() - q.n_state_aggs as usize..];
        let mut run = || -> GpuResult<()> {
            self.check(unsafe { sys::tskvgpu_scan_run(self.ctx, scan) })?;
            self.check(unsafe { sys::tskvgpu_scan_finalize(self.ctx, scan, values.as_mut_ptr(), validity.as_mut_ptr()) })?;
            for k in 0..q.n_state_aggs {
                maps.push(self.state_durations(scan, k, layout.n_cells)?);
                periods.push(if ops[k as usize].agg_mask as u32 == sys::TSKV_STATE_PERIODS {
                    Some(self.state_periods(scan, k, layout.n_cells)?)
                } else {
                    None
                });
            }
            Ok(())
        };
        let r = run();
        unsafe { sys::tskvgpu_scan_destroy(self.ctx, scan) };
        r.map(|_| (AggregateResult { layout, values, validity }, maps, periods))
    }

    /// The periods of state agg k (an operand with TSKV_STATE_PERIODS) of a scan that has run: sized by a first call
    /// with null arrays, then filled.
    fn state_periods(&self, scan: *mut sys::tskv_scan, k: u32, n_cells: u64) -> GpuResult<StatePeriods> {
        let mut n = 0u64;
        self.check(unsafe {
            sys::tskvgpu_scan_state_periods(self.ctx, scan, k, std::ptr::null_mut(), std::ptr::null_mut(), std::ptr::null_mut(),
                                            std::ptr::null_mut(), std::ptr::null_mut(), &mut n)
        })?;
        let mut p = StatePeriods {
            offsets: vec![0; n_cells as usize + 1],
            states: vec![0; n as usize],
            state_valid: vec![0; n as usize],
            starts: vec![0; n as usize],
            ends: vec![0; n as usize],
        };
        self.check(unsafe {
            sys::tskvgpu_scan_state_periods(self.ctx, scan, k, p.offsets.as_mut_ptr(), p.states.as_mut_ptr(), p.state_valid.as_mut_ptr(),
                                            p.starts.as_mut_ptr(), p.ends.as_mut_ptr(), &mut n)
        })?;
        Ok(p)
    }

    /// The maps of state agg k of a scan that has run: sized by a first call with null arrays, then filled.
    fn state_durations(&self, scan: *mut sys::tskv_scan, k: u32, n_cells: u64) -> GpuResult<StateDurations> {
        let mut n = 0u64;
        self.check(unsafe {
            sys::tskvgpu_scan_state_durations(self.ctx, scan, k, std::ptr::null_mut(), std::ptr::null_mut(), std::ptr::null_mut(),
                                              std::ptr::null_mut(), &mut n)
        })?;
        let mut m = StateDurations {
            offsets: vec![0; n_cells as usize + 1],
            states: vec![0; n as usize],
            state_valid: vec![0; n as usize],
            durations: vec![0; n as usize],
        };
        self.check(unsafe {
            sys::tskvgpu_scan_state_durations(self.ctx, scan, k, m.offsets.as_mut_ptr(), m.states.as_mut_ptr(),
                                              m.state_valid.as_mut_ptr(), m.durations.as_mut_ptr(), &mut n)
        })?;
        Ok(m)
    }

    fn output_layout(&self, pages: &PageSet<'_>, q: &Query, raw: &sys::tskv_query) -> GpuResult<sys::tskv_output_layout> {
        let mut layout = sys::tskv_output_layout::default();
        self.check(unsafe {
            match &q.groups {
                Some((ids, n)) => sys::tskvgpu_query_output_layout_grouped(pages.pages, raw, ids.as_ptr(), *n, &mut layout),
                None => sys::tskvgpu_query_output_layout(pages.pages, raw, &mut layout),
            }
        })?;
        Ok(layout)
    }

    /// Multi-GPU: this engine's rank in an NCCL communicator (collective: every rank calls it with rank 0's id).
    pub fn comm_init(&self, unique_id: &[u8; sys::TSKV_NCCL_UNIQUE_ID_BYTES], rank: i32, n_ranks: i32) -> GpuResult<()> {
        self.check(unsafe { sys::tskvgpu_comm_init(self.ctx, unique_id.as_ptr(), rank, n_ranks) })
    }

    /// Sharded scan: every rank scans its own pages with the GLOBAL series list (`Query::multi_rank`), exchanges the
    /// partial state with one ncclAllGather inside the library and finalises the merged result.
    pub fn scan_aggregate_sharded(&self, pages: &PageSet<'_>, q: &Query) -> GpuResult<AggregateResult> {
        let raw = q.as_raw()?;
        let layout = self.output_layout(pages, q, &raw)?;
        let mut scan = std::ptr::null_mut();
        self.check(unsafe {
            match (&q.groups, q.slide) {
                (Some((ids, n)), slide) => {
                    sys::tskvgpu_scan_prepare_grouped(self.ctx, pages.pages, &raw, ids.as_ptr(), *n, slide.unwrap_or(0), &mut scan)
                }
                (None, None) => sys::tskvgpu_scan_prepare(self.ctx, pages.pages, &raw, &mut scan),
                (None, Some(slide)) => sys::tskvgpu_scan_prepare_sliding(self.ctx, pages.pages, &raw, slide, &mut scan),
            }
        })?;
        let mut values = vec![0u64; (layout.n_out * layout.n_cells) as usize];
        let mut validity = vec![0u8; layout.validity_bytes as usize];
        let mut run = || -> GpuResult<()> {
            self.check(unsafe { sys::tskvgpu_scan_enqueue(self.ctx, scan) })?;
            self.check(unsafe { sys::tskvgpu_scan_exchange(self.ctx, scan) })?;
            self.check(unsafe { sys::tskvgpu_scan_finalize(self.ctx, scan, values.as_mut_ptr(), validity.as_mut_ptr()) })?;
            self.check(unsafe { sys::tskvgpu_scan_sync(self.ctx, scan) })
        };
        let r = run();
        unsafe { sys::tskvgpu_scan_destroy(self.ctx, scan) };
        r.map(|_| AggregateResult { layout, values, validity })
    }
}

impl Drop for GpuEngine {
    fn drop(&mut self) {
        unsafe { sys::tskvgpu_ctx_destroy(self.ctx) }
    }
}

/// rank 0: the 128 bytes the other ranks need for `GpuEngine::comm_init`.
pub fn comm_unique_id() -> GpuResult<[u8; sys::TSKV_NCCL_UNIQUE_ID_BYTES]> {
    let mut id = [0u8; sys::TSKV_NCCL_UNIQUE_ID_BYTES];
    match unsafe { sys::tskvgpu_comm_unique_id(id.as_mut_ptr()) } {
        sys::TSKV_OK => Ok(id),
        st => Err(GpuError { status: st, message: "libnccl.so.2 unavailable".into(), page: -1 }),
    }
}

/// A page arena known to the device (the engine's view of a cached `TsmReader`).
pub struct PageSet<'a> {
    engine: Arc<GpuEngine>,
    pages: *mut sys::tskv_pages,
    _arena: PhantomData<&'a [u8]>,
}
unsafe impl Send for PageSet<'_> {}
unsafe impl Sync for PageSet<'_> {}

impl PageSet<'_> {
    /// `ColumnGroup::time_range()` of every column group, in descriptor order: lets scans skip whole groups
    /// (`filter_column_groups`, tskv/src/reader/chunk.rs:12-50).
    pub fn set_time_bounds(&mut self, bounds: &[tskv_time_range]) -> GpuResult<()> {
        let st = unsafe { sys::tskvgpu_pages_set_time_bounds(self.engine.ctx, self.pages, bounds.as_ptr(), bounds.len() as u64) };
        self.engine.check(st)
    }
    /// The file's `TsmTombstone` cache flattened (tskv/src/tsm/tombstone.rs:417-550): one entry per excluded range.
    pub fn set_tombstones(&mut self, tombs: &[tskv_tombstone]) -> GpuResult<()> {
        let st = unsafe { sys::tskvgpu_pages_set_tombstones(self.engine.ctx, self.pages, tombs.as_ptr(), tombs.len() as u64) };
        self.engine.check(st)
    }
    /// `PageWriteSpec.meta.statistics` of every page, in descriptor order (`reader/column_group/statistics.rs:11-80`
    /// reads the same numbers): scans with field predicates skip the column groups the bounds rule out.
    pub fn set_value_stats(&mut self, stats: &[sys::tskv_value_stats]) -> GpuResult<()> {
        let st = unsafe { sys::tskvgpu_pages_set_value_stats(self.engine.ctx, self.pages, stats.as_ptr(), stats.len() as u64) };
        self.engine.check(st)
    }
    /// `ColumnFile::file_id()` (or the memcache's file id) of every column group, in descriptor order: scans merge
    /// the chunks of a series whose time ranges overlap, the newest file's non-null value winning per column
    /// (`DataMerger`, `reader/merge.rs`; `build_series_reader`, `reader/iterator.rs:463-560`).
    pub fn set_chunk_files(&mut self, cg_file_ids: &[u64]) -> GpuResult<()> {
        let st = unsafe { sys::tskvgpu_pages_set_chunk_files(self.engine.ctx, self.pages, cg_file_ids.as_ptr(), cg_file_ids.len() as u64) };
        self.engine.check(st)
    }
    pub fn series_count(&self) -> u64 {
        unsafe { sys::tskvgpu_pages_series_count(self.pages) }
    }
}

impl Drop for PageSet<'_> {
    fn drop(&mut self) {
        unsafe { sys::tskvgpu_pages_destroy(self.engine.ctx, self.pages) }
    }
}

/// The pushed-down scan: what `QueryOption` (tskv/src/reader/iterator.rs:713-741) carries for this path plus the
/// bucket expression and aggregate list that run in DataFusion today.
#[derive(Clone, Debug, Default)]
pub struct Query {
    /// sorted, unique (`get_series_id_by_filter`, tskv/src/kvcore.rs:249-279); `None` = every series of the page set
    pub series_ids: Option<Vec<u32>>,
    pub time_ranges: Vec<tskv_time_range>,
    pub origin: i64,
    /// bucket width in the time column's unit; <= 0: no bucketing. With `slide`: the window length
    pub width: i64,
    pub first_bucket_start: i64,
    pub n_buckets: u32,
    /// `time_window(time, width, slide, origin)`: output bucket j is the window starting at
    /// `first_bucket_start + j * slide`; `None` = tumbling buckets of `width`
    pub slide: Option<i64>,
    pub group_by_series: bool,
    /// GROUP BY tags: (group id of every selected series slot, number of groups); output cell = group * n_buckets +
    /// bucket. The shim derives dense ids from the `SeriesKey` tag values (INTEGRATION.md section 6).
    pub groups: Option<(Vec<u32>, u32)>,
    /// the projected columns, then the `n_gauges` gauges' operands, then the `n_state_aggs` state aggs' operands
    /// (agg_mask 0)
    pub columns: Vec<tskv_agg_column>,
    pub predicates: Vec<tskv_field_predicate>,
    pub multi_rank: bool,
    /// gauge_agg(time, x): the last `n_gauges` entries of `columns` are the operands (at most TSKV_MAX_GAUGES); each adds
    /// 9 outputs after the projected columns' (n, then t / v of the first, second, penultimate and last point), from
    /// which the shim builds DataFusion's GaugeData struct column (INTEGRATION.md section 6)
    pub n_gauges: u32,
    /// compact_state_agg(time, x): the last `n_state_aggs` entries of `columns` are the operands (I64 / U64, at most
    /// TSKV_MAX_STATE_AGGS); each adds 1 output after the gauges' (the cell's map entries), and
    /// `GpuEngine::scan_aggregate_states` returns the maps, from which the shim builds the DurationStates list column
    /// (INTEGRATION.md section 6); an operand with agg_mask TSKV_STATE_PERIODS (state_agg(time, x)) returns its
    /// periods too
    pub n_state_aggs: u32,
}

/// One state agg's maps in CSR form (tskvgpu_scan_state_durations): cell c owns entries `offsets[c]..offsets[c + 1]`,
/// the NULL state (`state_valid` 0) first, then the states (i64 / u64 bit patterns) in the type's order; `durations` in
/// the time column's unit.
#[derive(Clone, Debug, Default)]
pub struct StateDurations {
    pub offsets: Vec<u64>,
    pub states: Vec<u64>,
    pub state_valid: Vec<u8>,
    pub durations: Vec<i64>,
}

/// One state agg's periods in CSR form (tskvgpu_scan_state_periods): cell c owns periods `offsets[c]..offsets[c + 1]`,
/// the NULL state (`state_valid` 0) first, then the states (i64 / u64 bit patterns) in the type's order, each state's
/// maximal periods `[starts[i], ends[i])` by start, in the time column's unit. The shim builds state_agg's
/// `state_periods` list column from them (INTEGRATION.md section 6).
#[derive(Clone, Debug, Default)]
pub struct StatePeriods {
    pub offsets: Vec<u64>,
    pub states: Vec<u64>,
    pub state_valid: Vec<u8>,
    pub starts: Vec<i64>,
    pub ends: Vec<i64>,
}

impl Query {
    /// The C view of the query; TSKV_ERR_INVALID_ARG when `n_gauges` exceeds TSKV_MAX_GAUGES, `n_state_aggs`
    /// TSKV_MAX_STATE_AGGS, or their sum the entries of `columns` (the library would read operands past the Vec).
    fn as_raw(&self) -> GpuResult<sys::tskv_query> {
        let n_ops = self.n_gauges as usize + self.n_state_aggs as usize;
        if self.n_gauges > sys::TSKV_MAX_GAUGES || self.n_state_aggs > sys::TSKV_MAX_STATE_AGGS || n_ops > self.columns.len() {
            return Err(GpuError {
                status: sys::TSKV_ERR_INVALID_ARG,
                message: format!("n_gauges {} / n_state_aggs {} exceed their maxima or the {} column entries", self.n_gauges,
                                 self.n_state_aggs, self.columns.len()),
                page: -1,
            });
        }
        Ok(sys::tskv_query {
            series_ids: self.series_ids.as_ref().map_or(std::ptr::null(), |v| v.as_ptr()),
            n_series: self.series_ids.as_ref().map_or(0, |v| v.len() as u32),
            n_time_ranges: self.time_ranges.len() as u32,
            time_ranges: self.time_ranges.as_ptr(),
            origin: self.origin,
            width: self.width,
            first_bucket_start: self.first_bucket_start,
            n_buckets: self.n_buckets.max(1),
            group_by_series: self.group_by_series as u32,
            columns: self.columns.as_ptr(),
            n_columns: (self.columns.len() - n_ops) as u32,
            reserved: (if self.multi_rank { sys::TSKV_QUERY_MULTI_RANK } else { 0 })
                | sys::tskv_query_gauges(self.n_gauges)
                | sys::tskv_query_state_aggs(self.n_state_aggs),
            predicates: if self.predicates.is_empty() { std::ptr::null() } else { self.predicates.as_ptr() },
            n_predicates: self.predicates.len() as u32,
            n_pairs: 0,
        })
    }
}

/// Dense result, Arrow-compatible: output column j (query columns in order, aggregates in ascending bit order), cell
/// c = group * n_buckets + bucket: `values[j * n_cells + c]`, validity bit `c` of `validity[j * bitmap_stride ..]`
/// (LSB first). The `BatchReader` wraps both buffers as Arrow arrays without copying.
pub struct AggregateResult {
    pub layout: sys::tskv_output_layout,
    pub values: Vec<u64>,
    pub validity: Vec<u8>,
}

impl AggregateResult {
    pub fn value(&self, out_col: usize, cell: usize) -> Option<u64> {
        let stride = self.layout.bitmap_stride as usize;
        let valid = (self.validity[out_col * stride + (cell >> 3)] >> (cell & 7)) & 1 == 1;
        valid.then(|| self.values[out_col * self.layout.n_cells as usize + cell])
    }
}
