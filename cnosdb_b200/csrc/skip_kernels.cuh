// skip_kernels.cuh — builds the restart points ("skip index") of a page set, once, when the pages are uploaded.
//
// The reference decodes a page from its first byte every time (tskv/src/tsm/codec/{timestamp,integer,float}.rs): on
// a CPU a page is one core's work anyway. Here one page's serial stream is the longest dependent chain of a scan, so
// the page set keeps the decoder state at every SKIP_ROWS-th row of every simple8b / gorilla page (SkipEntry,
// cursors.cuh) - an acceleration structure over immutable pages, like the per-page statistics the reference keeps in
// PageMeta - and the fused scan enters a page at any of them. The builder IS the scan's own cursors (same structs,
// same staging rings): an entry is a snapshot of their state, so a restarted cursor continues bit-identically.
// A page whose stream does not decode cleanly up to its last restart point gets none (skip_off = SKIP_NONE): the scan
// then reads it from the start and reports the reference's error for it.
#pragma once
#include "cursors.cuh"

namespace tskv {

enum { SKIP_KIND_TIME_S8B = 0, SKIP_KIND_VALUE_S8B = 1, SKIP_KIND_VALUE_GORILLA = 2 };
constexpr int SKIP_THREADS = 128;
constexpr uint32_t SKIP_SMEM_BYTES = (SKIP_THREADS / 32) * RING_BYTES_PER_WARP;

// One lane per page of `page_list` (pages of one kind). Restart points for the pages with skip_off[page] != SKIP_NONE
// (more than SKIP_ROWS rows; skip_off null: none). KIND == SKIP_KIND_VALUE_S8B also decodes every value of the page and
// sets narrow[page] = 1 when each one lies in [-2^31, 2^31) (i64) or [0, 2^31) (u64) and the stream holds them all (the
// fused scan then accumulates the page in 32-bit arithmetic, ScanParams.page_narrow). A u64 value must not wrap to a
// negative i64: near 2^64 it sign-extends from 32 bits too, but its sums and order are unsigned.
template <int KIND>
__global__ void __launch_bounds__(SKIP_THREADS) k_build_skip(const uint8_t *arena, const tskv_page_desc *descs,
                                                             const uint32_t *page_list, uint32_t n_pages,
                                                             uint32_t *skip_off, SkipEntry *skip, uint8_t *narrow) {
  extern __shared__ __align__(16) uint8_t s_rings[];
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t slot = (uint32_t)__cvta_generic_to_shared(s_rings) + warp * RING_BYTES_PER_WARP + lane * RING_BYTES;
  const uint32_t i = blockIdx.x * SKIP_THREADS + threadIdx.x;
  const bool have = i < n_pages;
  uint32_t page = 0, n_rows = 0, page_rows = 0, off = SKIP_NONE;
  bool is_u64 = false;
  PageView pv;
  S8bCursor<KIND == SKIP_KIND_VALUE_S8B> sc;
  GorillaRing gc;
  if (KIND == SKIP_KIND_VALUE_GORILLA) gc.reset(slot);
  else sc.reset(slot);
  if (have) {
    page = page_list[i];
    const tskv_page_desc d = descs[page];
    if (skip_off) off = skip_off[page];
    pv.open(arena, d);
    page_rows = n_rows = d.num_values;
    is_u64 = d.phys_type == TSKV_PT_U64;
    if (KIND == SKIP_KIND_VALUE_GORILLA) gc.open(pv, slot);
    else sc.open(pv, d.reserved, slot);
  }
  ring_drain();
  if (!have || off == SKIP_NONE) n_rows = 0;
  const uint32_t n_entries = n_rows ? (n_rows - 1) / SKIP_ROWS : 0;
  const uint32_t *bm = reinterpret_cast<const uint32_t *>(pv.bitset);
  bool ok = true;
  if (KIND == SKIP_KIND_TIME_S8B) {
    // time pages hold no nulls (pages that do are never cut): entry j = the state after row j * SKIP_ROWS's timestamp
    const uint32_t last = n_entries * SKIP_ROWS;
    for (uint32_t r = 0; r <= last && n_entries; r++) {
      sc.next();
      if (r && (r % SKIP_ROWS) == 0) {
        if (sc.exhausted()) { ok = false; break; }
        skip[off + r / SKIP_ROWS - 1] = sc.save(pv);
      }
    }
  } else if (KIND == SKIP_KIND_VALUE_S8B) {
    // value pages: entry j = the state before the first value of a row >= j * SKIP_ROWS (only valid rows hold one);
    // the walk goes on to the page's last row for the narrow flag
    uint32_t word = 0;
    const uint32_t last = n_entries * SKIP_ROWS;
    bool nar = true;
    for (uint32_t r = 0; r < page_rows; r++) {
      if ((r & 31) == 0) word = __ldg(bm + (r >> 5));
      if (ok && r && r <= last && (r % SKIP_ROWS) == 0) {
        if (sc.exhausted()) ok = false;
        else skip[off + r / SKIP_ROWS - 1] = sc.save(pv);
      }
      if ((word >> (r & 31)) & 1) {
        const uint64_t v = sc.next();
        nar = nar && (is_u64 ? (v >> 31) == 0 : (int64_t)(int32_t)v == (int64_t)v);
      }
    }
    if (have) narrow[page] = (nar && !sc.exhausted()) ? 1 : 0;
  } else {
    uint32_t word = 0;
    const uint32_t last = n_entries * SKIP_ROWS;
    for (uint32_t r = 0; r <= last && n_entries; r++) {
      if ((r & 31) == 0) word = __ldg(bm + (r >> 5));
      if (r && (r % SKIP_ROWS) == 0) {
        if (gc.failed()) { ok = false; break; }
        skip[off + r / SKIP_ROWS - 1] = gc.save(pv);
        if (r == last) break;
      }
      if ((word >> (r & 31)) & 1) gc.next();
    }
  }
  if (have && off != SKIP_NONE && !ok) skip_off[page] = SKIP_NONE;
  ring_drain();
}

}  // namespace tskv
