// decode_kernels.cuh — decode-only path (Page::to_arrow_array / data_buf_to_arrow_array, tsm/reader.rs:658-731):
// values + Arrow validity bitmap of whole pages to HBM (BASELINE config C1, and the debugging / export path).
//
//   k_decode_warp   one WARP per page. Codecs whose values are independent given a prefix sum are decoded by
//                   the whole warp - simple8b words lane-per-word (coalesced 8-byte loads, selector lookup, warp
//                   exclusive scan of the counts for the output offsets, warp inclusive scan of the per-word delta
//                   sums for the running value), raw pages lane-per-value, RLE pages in closed form from the validity
//                   ranks - so a single long page (C1: one series x 10 000 points) uses 32 lanes and every store is to
//                   consecutive addresses. Pages that need a serial walk (gorilla: each value's position depends on
//                   the control bits before it; simple8b / raw pages WITH nulls: value k belongs to the k-th set bit)
//                   are decoded by lane 0 with the streaming cursors of cursors.cuh.
// Same formats and error classes as the fused scan (cursors.cuh cites the reference lines).
#pragma once
#include "scan_kernels.cuh"

namespace tskv {

// One page by one lane, row by row (the round-1 decode kernel's body).
__device__ inline tskv_status decode_page_serial(const uint8_t *arena, const tskv_page_desc &d, uint64_t *ov, uint32_t *ob,
                                                 unsigned long long *points_out) {
  tskv_status st = kind_status(d.reserved);
  const uint32_t n_rows = d.num_values;
  unsigned long long points = 0;
  if (st == TSKV_OK) {
    PageView pv;
    pv.open(arena, d);
    BitCursor bits;
    bits.init(pv.bitset);
    AnyCursor<> cur;
    st = cur.open(pv, d.reserved);
    const bool allnull = d.reserved == DK_ALLNULL;
    uint32_t wbits = 0;
    for (uint32_t r = 0; r < n_rows && st == TSKV_OK; r++) {
      bool valid = bits.next(r) && !allnull;
      uint64_t v = 0;
      if (valid) {
        v = cur.next();
        if (cur.failed()) { st = cur.stream_error() ? TSKV_ERR_SHORT_BLOCK : TSKV_ERR_BITSET_MISMATCH; break; }
        points++;
      } else if (r == 0 && !cur.is_gorilla) {
        cur.d.skip_first_if_s8b_sc();
      }
      ov[r] = v;
      wbits |= (valid ? 1u : 0u) << (r & 31);
      if ((r & 31) == 31) { ob[r >> 5] = wbits; wbits = 0; }
    }
    if (st == TSKV_OK) {
      if (n_rows & 31) ob[n_rows >> 5] = wbits;
      // zero the tail of the 8-byte-padded bitmap
      uint32_t words = ((n_rows + 63) / 64) * 2;
      for (uint32_t w = (n_rows + 31) / 32; w < words; w++) ob[w] = 0;
      if (cur.is_gorilla && cur.g.consumed_any() && !cur.g.drain()) st = TSKV_ERR_SHORT_BLOCK;
    }
  }
  *points_out = points;
  return st;
}

__device__ __forceinline__ uint64_t load_be64_any(const uint8_t *p) {
  const uintptr_t a = reinterpret_cast<uintptr_t>(p);
  const uint64_t *ap = reinterpret_cast<const uint64_t *>(a & ~(uintptr_t)7);
  const uint32_t sh = (uint32_t)(a & 7) * 8;
  const uint64_t lo = __ldg(ap), hi = __ldg(ap + 1);
  return bswap64((lo >> sh) | ((hi << 1) << (63 - sh)));
}

__device__ __forceinline__ uint32_t warp_excl_scan_u32(uint32_t v, uint32_t *total) {
  const uint32_t lane = threadIdx.x & 31;
  uint32_t x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t y = __shfl_up_sync(FULL, x, o);
    if (lane >= (uint32_t)o) x += y;
  }
  *total = __shfl_sync(FULL, x, 31);
  return x - v;
}
__device__ __forceinline__ uint64_t warp_incl_scan_u64(uint64_t v) {
  const uint32_t lane = threadIdx.x & 31;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t lo = __shfl_up_sync(FULL, (uint32_t)v, o), hi = __shfl_up_sync(FULL, (uint32_t)(v >> 32), o);
    if (lane >= (uint32_t)o) v += ((uint64_t)hi << 32) | lo;
  }
  return v;
}

// Cooperative simple8b delta decode straight to global memory: dst[i] = first + sum_{j<=i} d(u_j) for i < cap.
// Returns how many values the stream holds (first value included).
template <bool ZZ>
__device__ __forceinline__ uint64_t decode_s8b_to_global(const uint8_t *words, uint32_t n_words, uint64_t first,
                                                         uint64_t scaler, uint64_t *dst, uint32_t cap) {
  const uint32_t lane = threadIdx.x & 31;
  if (lane == 0 && cap) dst[0] = first;
  uint64_t carry = first;
  uint64_t base = 1;
  for (uint32_t w0 = 0; w0 < n_words; w0 += 32) {
    const uint32_t wi = w0 + lane;
    const bool have = wi < n_words;
    const uint64_t word = have ? load_be64_any(words + 8ull * wi) : 0;
    const uint32_t sel = (uint32_t)(word >> 60);
    uint32_t cnt, bits;
    s8b_lut(sel, cnt, bits);
    if (!have) cnt = 0;
    const uint64_t mask = bits ? (~0ull >> (64 - bits)) : 0ull;
    uint32_t total;
    const uint64_t pos = base + warp_excl_scan_u32(cnt, &total);
    uint64_t wsum = 0;  // pass 1: sum of this word's deltas
    if (sel < 2) {
      wsum = (ZZ ? (uint64_t)zigzag_dec(1) : scaler) * cnt;
    } else {
      uint64_t x = word & 0x0fffffffffffffffull;
      for (uint32_t k = 0; k < cnt; k++) {
        const uint64_t u = x & mask;
        x >>= bits;
        wsum += ZZ ? (uint64_t)zigzag_dec(u) : u * scaler;
      }
    }
    const uint64_t incl = warp_incl_scan_u64(wsum);
    uint64_t run = carry + incl - wsum;
    uint64_t x = word & 0x0fffffffffffffffull;  // pass 2: running prefix to the output
    for (uint32_t k = 0; k < cnt; k++) {
      const uint64_t u = sel < 2 ? 1ull : (x & mask);
      x >>= bits;
      run += ZZ ? (uint64_t)zigzag_dec(u) : u * scaler;
      if (pos + k < cap) dst[pos + k] = run;
    }
    carry += shfl_u64(incl, 31);
    base += total;
  }
  return base;
}

constexpr int DECODE_THREADS = 128;

__global__ void __launch_bounds__(DECODE_THREADS)
k_decode_warp(const uint8_t *arena, const tskv_page_desc *descs, uint64_t first_page, const uint32_t *page_list, uint32_t n_pages,
              const uint64_t *row_off, const uint64_t *bm_off, uint64_t *out_values, uint8_t *out_validity,
              int32_t *status, unsigned long long *err_page, unsigned long long *stats) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (i >= n_pages) return;
  const uint32_t page = page_list ? page_list[i] : (uint32_t)first_page + i;  // a page range, or a list of pages
  const tskv_page_desc d = descs[page];
  uint64_t *ov = out_values + row_off[i];
  uint32_t *ob = reinterpret_cast<uint32_t *>(out_validity + bm_off[i]);
  const uint32_t n_rows = d.num_values;
  tskv_status st = kind_status(d.reserved);
  unsigned long long points = 0;
  if (st == TSKV_OK) {
    PageView pv;
    pv.open(arena, d);
    const uint8_t kind = d.reserved;
    // validity bitmap -> output (8-byte padded), and: does the page hold nulls?
    const uint32_t *bm = reinterpret_cast<const uint32_t *>(pv.bitset);
    const uint32_t n_bm = (n_rows + 31) >> 5, out_words = ((n_rows + 63) / 64) * 2;
    bool full = true;
    uint32_t valid_rows = 0;
    for (uint32_t w = lane; w < out_words; w += 32) {
      uint32_t bits = 0;
      if (w < n_bm && kind != DK_ALLNULL) {
        bits = __ldg(bm + w);
        const uint32_t want = (w == n_bm - 1 && (n_rows & 31)) ? ((1u << (n_rows & 31)) - 1) : 0xffffffffu;
        bits &= want;
        full = full && bits == want;
      }
      ob[w] = bits;
      valid_rows += __popc(bits);
    }
    full = __all_sync(FULL, full);
    valid_rows = __reduce_add_sync(FULL, valid_rows);
    const uint8_t *dd = pv.data;
    bool serial = false;
    switch (kind) {
      case DK_ALLNULL:
        break;  // the output values were zeroed by the host
      case DK_RLE_SC:    // timestamp.rs:226-259
      case DK_RLE_ZZ: {  // integer.rs:186-214
        uint64_t dl = 0;
        if (!decode_varint(dd + 10, pv.data_len - 10, &dl)) { st = TSKV_ERR_SHORT_BLOCK; break; }
        const uint64_t delta = kind == DK_RLE_SC ? dl * pow10_u64(__ldg(dd + 1) & 0xf) : (uint64_t)zigzag_dec(dl);
        const uint64_t first = kind == DK_RLE_SC ? load_be64_any(dd + 2) : (uint64_t)zigzag_dec(load_be64_any(dd + 2));
        uint32_t rank_base = 0;  // the k-th VALID row holds first + k * delta
        for (uint32_t r0 = 0; r0 < n_rows; r0 += 32) {
          uint32_t bits = __ldg(bm + (r0 >> 5));
          if (n_rows - r0 < 32) bits &= (1u << (n_rows - r0)) - 1;
          const uint32_t r = r0 + lane;
          if (r < n_rows) {
            const bool v = (bits >> lane) & 1;
            ov[r] = v ? first + (uint64_t)(rank_base + __popc(bits & ((1u << lane) - 1))) * delta : 0ull;
          }
          rank_base += __popc(bits);
        }
        points = valid_rows;
        break;
      }
      case DK_S8B_SC:    // timestamp.rs:261-299
      case DK_S8B_ZZ: {  // integer.rs:216-248
        if (!full) { serial = true; break; }
        const uint64_t scaler = kind == DK_S8B_SC ? pow10_u64(__ldg(dd + 1) & 0xf) : 1;
        const uint64_t first = kind == DK_S8B_SC ? load_be64_any(dd + 2) : (uint64_t)zigzag_dec(load_be64_any(dd + 2));
        const uint64_t got = kind == DK_S8B_SC
                                 ? decode_s8b_to_global<false>(dd + 10, (pv.data_len - 10) >> 3, first, scaler, ov, n_rows)
                                 : decode_s8b_to_global<true>(dd + 10, (pv.data_len - 10) >> 3, first, scaler, ov, n_rows);
        if (got < n_rows) st = TSKV_ERR_BITSET_MISMATCH;
        points = n_rows;
        break;
      }
      case DK_RAW_SC:    // timestamp.rs:201-224: prefix sum of 8-byte BE deltas
      case DK_RAW_ZZ:    // integer.rs:165-184
      case DK_RAWBE: {   // timestamp.rs:301-323, float.rs:387-413
        if (!full) { serial = true; break; }
        const uint8_t *w = dd + (kind == DK_RAWBE ? 1 : 2);
        const uint32_t n_words = (pv.data_len - (kind == DK_RAWBE ? 1 : 2)) >> 3;
        if (n_words < n_rows) { st = TSKV_ERR_BITSET_MISMATCH; break; }
        uint64_t carry = 0;
        for (uint32_t r0 = 0; r0 < n_rows; r0 += 32) {
          const uint32_t r = r0 + lane;
          uint64_t v = r < n_rows ? load_be64_any(w + 8ull * r) : 0;
          if (kind == DK_RAW_ZZ) v = (uint64_t)zigzag_dec(v);
          if (kind != DK_RAWBE) {
            v = warp_incl_scan_u64(v) + carry;
            carry = shfl_u64(v, 31);
          }
          if (r < n_rows) ov[r] = v;
        }
        points = n_rows;
        break;
      }
      default:  // gorilla: a serial walk
        serial = true;
        break;
    }
    if (serial) {
      unsigned long long p = 0;
      int s2 = TSKV_OK;
      if (lane == 0) s2 = decode_page_serial(arena, d, ov, ob, &p);
      st = (tskv_status)__shfl_sync(FULL, s2, 0);
      points = p;  // lane 0's count is the page's
    }
  }
  if (lane == 0) {
    if (st != TSKV_OK && atomicCAS(status, 0, (int)st) == 0) *err_page = page;
    if (points) atomicAdd(&stats[0], points);
  }
}

// Value statistics of every field page (what the reference keeps in PageMeta.statistics, tsm/page.rs:599-613): min / max
// of the non-null (f64: non-NaN) values as ordered keys (stats_key, scan_kernels.cuh), once per page set, for the
// value-statistics pruning of scans with field predicates. One lane per page, the serial cursors.
__global__ void k_page_stats(const uint8_t *arena, const tskv_page_desc *descs, uint64_t n_descs, int64_t *stats) {
  const uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n_descs) return;
  const tskv_page_desc d = descs[p];
  int64_t kmin = INT64_MAX, kmax = INT64_MIN;
  bool ok = d.phys_type != TSKV_PT_TIME && kind_status(d.reserved) == TSKV_OK;
  if (ok) {
    PageView pv;
    pv.open(arena, d);
    BitCursor bits;
    bits.init(pv.bitset);
    AnyCursor<> cur;
    ok = cur.open(pv, d.reserved) == TSKV_OK;
    const bool allnull = d.reserved == DK_ALLNULL;
    for (uint32_t r = 0; r < d.num_values && ok; r++) {
      if (bits.next(r) && !allnull) {
        const uint64_t v = cur.next();
        if (cur.failed()) { ok = false; break; }
        if (d.phys_type == TSKV_PT_F64 && (v & 0x7fffffffffffffffull) > 0x7ff0000000000000ull) continue;  // NaN: never TRUE
        const int64_t k = stats_key(v, d.phys_type);
        kmin = k < kmin ? k : kmin;
        kmax = k > kmax ? k : kmax;
      } else if (r == 0 && !cur.is_gorilla) {
        cur.d.skip_first_if_s8b_sc();
      }
    }
  }
  if (!ok) { kmin = INT64_MIN; kmax = INT64_MAX; }  // unknown: nothing can be ruled out
  stats[2 * p] = kmin;
  stats[2 * p + 1] = kmax;
}

}  // namespace tskv
