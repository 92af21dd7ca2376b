// coop_kernels.cuh — warp-cooperative scan of ONE page per warp (sm_90a), for the codecs that decode in
// parallel: timestamps RLE / simple8b, values zig-zag simple8b — and, split in two phases, gorilla values.
//
// The lane-per-page kernels (scan_kernels.cuh) are bounded by the serial decode latency of one page
// (1000 rows x ~120 dependent instructions) no matter how many SMs or GPUs share the work. Here a warp
//   A. decodes the time page into shared memory (skipped for RLE: closed form),
//   B. decodes the value page into shared memory: 32 simple8b words per step with coalesced 8-byte loads,
//      selector -> count LUT, warp exclusive scan for the output offsets, unpack, warp inclusive scan of the
//      per-word delta sums for the running prefix (the carry crosses steps),
//   C. computes per row (lane-per-row) the (selected, bucket) key with a multiply-high division by the
//      invariant bucket width and compacts the segment heads,
//   D. reduces lane-per-segment (a 1-minute bucket of a 10-second series is 6 rows) and updates the
//      per-CTA shared-memory table / the global state once per segment and aggregate.
// Gorilla (float.rs:418-606) is bit-serial only in its STRUCTURE (where each value's XOR window starts depends on
// the control bits before it), so its pages are decoded in two phases by the same warp, a group of G pages at a time:
//   1. lane g parses the control bits of page g (13 bits per element, ~20 dependent instructions) and writes one
//      32-bit record per element {mantissa bit offset, meaningful bits, trailing zeros} to a global scratch row;
//   2. the warp takes the G pages one by one: lane-per-value mantissa extraction from the records, a warp XOR scan
//      for the running value, then steps C and D as for the integer pages.
// G is chosen by the host so that the selected pages make about one task per resident warp.
// Same formats and semantics as cursors.cuh / scan_kernels.cuh (reference lines cited there).
#pragma once
#include <cstddef>

#include "scan_kernels.cuh"

namespace tskv {

constexpr int COOP_TILE = 1024;              // pages with more rows use the lane-per-page kernels
constexpr int COOP_PAD = COOP_TILE + COOP_TILE / 32 + 8;
__host__ __device__ __forceinline__ uint32_t cpad(uint32_t i) { return i + (i >> 5); }

constexpr uint32_t GOR_REC_STRIDE = COOP_TILE + 8;  // u32 records per page row in the scratch
constexpr uint64_t GOR_SENTINEL = 0x7ff80000000000ffull;  // float.rs:16

// Phase-1 result of one gorilla page (lane g of the group wrote entry g).
struct GorGroup {
  uint32_t n_valid[32];   // valid rows = values the bitset asks for
  uint32_t n_parsed[32];  // elements 1..n_parsed parsed inside the block (< n_valid: element n_parsed + 1 overran it)
  uint32_t endpos[32];    // stream bit position after the last parsed element
  uint8_t meaningful[32], trailing[32];  // window state after the last parsed element
};

struct NoGorGroup {};
template <bool GOR> struct GorGroupSel { using type = GorGroup; };
template <> struct GorGroupSel<false> { using type = NoGorGroup; };

template <bool HAS_TS, bool GOR>
struct CoopSmem {
  uint64_t vals[COOP_PAD];
  uint64_t ts[HAS_TS ? COOP_PAD : 1];
  uint16_t seg[COOP_TILE + 2];
  uint32_t rank_base[COOP_TILE / 32 + 1];
  typename GorGroupSel<GOR>::type gor;
};

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
__device__ __forceinline__ uint64_t warp_incl_xor_scan_u64(uint64_t v) {
  const uint32_t lane = threadIdx.x & 31;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t lo = __shfl_up_sync(FULL, (uint32_t)v, o), hi = __shfl_up_sync(FULL, (uint32_t)(v >> 32), o);
    if (lane >= (uint32_t)o) v ^= ((uint64_t)hi << 32) | lo;
  }
  return v;
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

// Cooperative simple8b delta decode (simple8b.rs:80-208 + timestamp.rs:261-299 / integer.rs:216-248):
// dst[cpad(i)] = first + sum_{j<=i} d(u_j), d = zig-zag decode (ZZ) or u * scaler. Writes at most `cap`
// values; returns how many values the stream holds (first value included).
template <bool ZZ>
__device__ __forceinline__ uint32_t coop_decode_s8b(const uint8_t *words, uint32_t n_words, uint64_t first,
                                                    uint64_t scaler, uint64_t *dst, uint32_t cap) {
  const uint32_t lane = threadIdx.x & 31;
  if (lane == 0 && cap) dst[0] = first;
  uint64_t carry = first;
  uint32_t base = 1;
  for (uint32_t w0 = 0; w0 < n_words; w0 += 32) {
    const uint32_t wi = w0 + lane;
    const bool have = wi < n_words;
    const uint64_t word = have ? load_be64_any(words + 8ull * wi) : 0;
    const uint32_t sel = (uint32_t)(word >> 60);
    const uint32_t cnt = have ? c_s8b_count[sel] : 0;
    const uint32_t bits = c_s8b_bits[sel];
    const uint64_t mask = bits ? (~0ull >> (64 - bits)) : 0ull;
    uint32_t total;
    const uint32_t pos = base + warp_excl_scan_u32(cnt, &total);
    // pass 1: sum of this word's deltas
    uint64_t wsum = 0;
    if (sel < 2) {
      const uint64_t one = ZZ ? (uint64_t)zigzag_dec(1) : scaler;
      wsum = one * cnt;
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
    // pass 2: running prefix to shared memory
    {
      uint64_t x = word & 0x0fffffffffffffffull;
      for (uint32_t k = 0; k < cnt; k++) {
        const uint64_t u = sel < 2 ? 1ull : (x & mask);
        x >>= bits;
        run += ZZ ? (uint64_t)zigzag_dec(u) : u * scaler;
        if (pos + k < cap) dst[cpad(pos + k)] = run;
      }
    }
    carry += shfl_u64(incl, 31);
    base += total;
  }
  return base;
}

// ---- gorilla, phase 1 and bit helpers -------------------------------------------------------------------------
// MSB-first bit stream addressed through 4-byte aligned words: `wp` = aligned pointer at or below the stream start,
// `abs` = bit offset from wp. Reads may run <= 12 bytes past the page (arena slack).
__device__ __forceinline__ uint32_t gor_peek32(const uint32_t *wp, uint32_t abs) {
  const uint32_t wi = abs >> 5;
  const uint32_t a = __byte_perm(__ldg(wp + wi), 0, 0x0123), b = __byte_perm(__ldg(wp + wi + 1), 0, 0x0123);
  return __funnelshift_l(b, a, abs & 31);
}
__device__ __forceinline__ uint64_t gor_peek64(const uint32_t *wp, uint32_t abs) {
  const uint32_t wi = abs >> 5, sh = abs & 31;
  const uint32_t a = __byte_perm(__ldg(wp + wi), 0, 0x0123), b = __byte_perm(__ldg(wp + wi + 1), 0, 0x0123),
                 c = __byte_perm(__ldg(wp + wi + 2), 0, 0x0123);
  return ((uint64_t)__funnelshift_l(b, a, sh) << 32) | __funnelshift_l(c, b, sh);
}
// One element's control bits (float.rs:480-560, cursors.cuh GorillaCursor::advance): returns the control length,
// sets `sig` = XOR-window width (0: repeat the previous value) and updates the (meaningful, trailing) window state.
__device__ __forceinline__ uint32_t gor_parse_ctrl(uint32_t x13, uint32_t &meaningful, uint32_t &trailing, uint32_t &sig) {
  // branch-free: the lanes of a warp parse different pages and would diverge on every element
  const bool c0 = x13 & 0x1000, c1 = x13 & 0x0800;
  const uint32_t leading = (x13 >> 6) & 0x1f, m = x13 & 0x3f;
  const uint32_t new_mean = m ? m : 64u;
  const uint32_t new_trail = m ? ((64u - leading - m) & 0xffu) : 0u;  // u8 arithmetic like the reference
  const bool fresh = c0 && c1;
  meaningful = fresh ? new_mean : meaningful;
  trailing = fresh ? new_trail : trailing;
  sig = c0 ? meaningful : 0u;
  return c0 ? (c1 ? 13u : 2u) : 1u;
}
__device__ __forceinline__ void gor_stream(const PageView &vpv, const uint32_t *&wp, uint32_t &base_bits, uint32_t &total_bits) {
  const uintptr_t a = reinterpret_cast<uintptr_t>(vpv.data + 10);  // id | 0x10 | first(8) | bit stream
  wp = reinterpret_cast<const uint32_t *>(a & ~(uintptr_t)3);
  base_bits = (uint32_t)(a & 3) * 8;
  total_bits = (vpv.data_len - 10) * 8;
}

// Phase 1, one lane per page: records[e] for the elements e = 1..n_valid (element n_valid is the one that has to be
// the sentinel); remembers the first element that runs past the block (n_parsed = the elements before it).
__device__ __forceinline__ void gor_parse_page(const ScanParams &P, uint32_t item, uint32_t *records, GorGroup &G, uint32_t g) {
  const uint32_t page = P.work_page[item];
  const tskv_page_desc vd = P.descs[page];
  PageView vpv;
  vpv.open(P.arena, vd);
  const uint32_t n_rows = vd.num_values;
  const uint32_t *vbm = reinterpret_cast<const uint32_t *>(vpv.bitset);
  uint32_t n_valid = 0;
  for (uint32_t w = 0; w < (n_rows + 31) >> 5; w++) {
    uint32_t bits = __ldg(vbm + w);
    if (w == (n_rows >> 5)) bits &= (1u << (n_rows & 31)) - 1;
    n_valid += __popc(bits);
  }
  const uint32_t *wp;
  uint32_t base_bits, total_bits;
  gor_stream(vpv, wp, base_bits, total_bits);
  uint32_t bitpos = 0, meaningful = 64, trailing = 0, e = 1, first_over = 0;
  const uint32_t last_word = (base_bits + total_bits) >> 5;  // prefetches stay inside the page
  asm volatile("prefetch.global.L1 [%0];" ::"l"(wp));
  asm volatile("prefetch.global.L1 [%0];" ::"l"(wp + min(32u, last_word)));
  asm volatile("prefetch.global.L1 [%0];" ::"l"(wp + min(64u, last_word)));
#pragma unroll 1
  for (; e <= n_valid; e++) {
    uint32_t sig;
    // the walk is one dependent chain: without this the chain stalls on a DRAM round trip at every new sector
    const uint32_t rp = base_bits + min(bitpos, total_bits);  // (after an overrun the walk goes on, reading at the block's end)
    asm volatile("prefetch.global.L1 [%0];" ::"l"(wp + min((rp >> 5) + 96, last_word)));
    const uint32_t len = gor_parse_ctrl(gor_peek32(wp, rp) >> 19, meaningful, trailing, sig);
    records[e] = (bitpos + len) | (sig << 17) | ((trailing & 63) << 24);
    bitpos += len + sig;
    // "unexpected end of block" (bits_used > bits_total in the serial cursor): remembered, not branched on - the
    // loop's back edge must not wait for the end of the dependent chain (the reads are clamped to the block's end).
    first_over = (bitpos > total_bits && first_over == 0) ? e : first_over;
  }
  if (first_over) e = first_over;
  G.n_valid[g] = n_valid;
  G.n_parsed[g] = e - 1;
  G.endpos[g] = bitpos;
  G.meaningful[g] = (uint8_t)meaningful;
  G.trailing[g] = (uint8_t)trailing;
}

// Phase 1 for a group of ONE page: the warp first copies the page's bit stream into its shared memory (byte-swapped
// words, coalesced), then lane 0 walks the control bits from there: the dependent chain per element is two LDS + ~12
// ALU operations instead of global-memory round trips. `stage` overlays the warp's CoopSmem (free until phase 2).
__device__ __forceinline__ void gor_parse_page_staged(const ScanParams &P, uint32_t item, uint32_t *records, GorGroup &G,
                                                      uint32_t *stage, uint32_t stage_words) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t page = P.work_page[item];
  const tskv_page_desc vd = P.descs[page];
  PageView vpv;
  vpv.open(P.arena, vd);
  const uint32_t *wp;
  uint32_t base_bits, total_bits;
  gor_stream(vpv, wp, base_bits, total_bits);
  const uint32_t n_words = ((base_bits + total_bits + 31) >> 5) + 2;  // + the look-ahead words of the last peek
  if (n_words > stage_words) {  // does not fit (cannot happen for <= 1024 reference-written rows): parse from global memory
    if (lane == 0) gor_parse_page(P, item, records, G, 0);
    return;
  }
  for (uint32_t w = lane; w < n_words; w += 32) stage[w] = __byte_perm(__ldg(wp + w), 0, 0x0123);
  const uint32_t n_rows = vd.num_values;
  const uint32_t *vbm = reinterpret_cast<const uint32_t *>(vpv.bitset);
  uint32_t bits = 0;
  if (lane < ((n_rows + 31) >> 5)) {
    bits = __ldg(vbm + lane);
    if (lane == (n_rows >> 5)) bits &= (1u << (n_rows & 31)) - 1;
  }
  const uint32_t n_valid = __reduce_add_sync(FULL, __popc(bits));
  __syncwarp();
  if (lane == 0) {
    uint32_t bitpos = 0, meaningful = 64, trailing = 0, e = 1;
#pragma unroll 1
    for (; e <= n_valid; e++) {
      const uint32_t abs = base_bits + bitpos, wi = abs >> 5;
      uint32_t sig;
      const uint32_t len = gor_parse_ctrl(__funnelshift_l(stage[wi + 1], stage[wi], abs & 31) >> 19, meaningful, trailing, sig);
      records[e] = (bitpos + len) | (sig << 17) | ((trailing & 63) << 24);
      bitpos += len + sig;
      if (bitpos > total_bits) break;
    }
    G.n_valid[0] = n_valid;
    G.n_parsed[0] = e - 1;
    G.endpos[0] = bitpos;
    G.meaningful[0] = (uint8_t)meaningful;
    G.trailing[0] = (uint8_t)trailing;
  }
}

// Multiply-high division of a non-negative dividend by the invariant bucket width (Granlund-Montgomery):
// q = floor(x / d) for d >= 1 with m = floor(2^64 (2^l - d) / d) + 1, l = ceil(log2 d).
struct MagicDiv {
  uint64_t m;
  uint32_t l;  // 0 => d == 1
};
__device__ __forceinline__ uint64_t magic_div(uint64_t x, MagicDiv md) {
  if (md.l == 0) return x;
  const uint64_t t = __umul64hi(md.m, x);
  return (((x - t) >> 1) + t) >> (md.l - 1);
}

struct CoopParams {
  MagicDiv div;        // by P.width
  int64_t q0;          // quotient of first_bucket_start: bucket idx = q(t) - q0
  uint32_t grid_ok;    // first_bucket_start lies on the bucket grid
  uint32_t gor_group;  // gorilla bins: pages per warp task (1..32)
  uint32_t *gor_scratch[2];  // per gorilla bin: [warps of the grid][gor_group][GOR_REC_STRIDE] element records
};

// (selected by the time ranges, bucket) of one timestamp as a 32-bit key; 0xffffffff = not selected.
__device__ __forceinline__ uint32_t coop_row_key(const ScanParams &P, const CoopParams &C, int64_t t, bool *range_err) {
  bool in = P.n_ranges == 0;
#pragma unroll 1
  for (uint32_t k = 0; k < P.n_ranges && !in; k++) in = t >= P.ranges[k].min_ts && t <= P.ranges[k].max_ts;
  if (!in) return 0xffffffffu;
  if (P.width <= 0) return 0;
  const int64_t dividend = (int64_t)((uint64_t)t - (uint64_t)P.origin_mod + (uint64_t)P.width);
  int64_t idx;
  if (dividend >= 0 && C.grid_ok) {
    idx = (int64_t)magic_div((uint64_t)dividend, C.div) - C.q0;
  } else {  // the reference's truncating-% regime (time_window.rs:184-198): exact slow path
    const int64_t start = (int64_t)((uint64_t)t - (uint64_t)(dividend % P.width));
    const int64_t diff = (int64_t)((uint64_t)start - (uint64_t)P.first_bucket_start);
    idx = (diff % P.width != 0) ? -1 : diff / P.width;
  }
  if (idx < 0 || idx >= (int64_t)P.n_buckets) {
    *range_err = true;
    return 0xffffffffu;
  }
  return (uint32_t)idx;
}

// One page per warp. TK in {TK_RLE, TK_S8B} (time page without nulls), VK = VK_S8B (zig-zag simple8b values) or
// VK_GOR (gorilla values; `records` / entry `g` of S.gor = phase 1's output for this page).
template <int TK, int VK, bool SEL>
__device__ __forceinline__ void scan_page_coop(const ScanParams &P, const CoopParams &C, uint32_t item,
                                               CoopSmem<TK == TK_S8B, VK == VK_GOR> &S, uint64_t *stab,
                                               const uint32_t *records = nullptr, uint32_t g = 0) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t page = P.work_page[item];
  const uint32_t slot = P.work_slot[item];
  const uint32_t qcol = P.work_qcol[item] & 0x7f;
  const tskv_page_desc vd = P.descs[page];
  const uint32_t tpage = P.time_page_of[page];
  const tskv_page_desc td = P.descs[tpage];
  const ColState &cs = P.cols[qcol];
  const uint8_t pt = cs.phys_type, mask = cs.agg_mask;
  const uint32_t n_rows = vd.num_values;
  PageView tpv, vpv;
  tpv.open(P.arena, td);
  vpv.open(P.arena, vd);

  // ---- A. timestamps --------------------------------------------------------------------------------
  uint64_t t_first = 0, t_delta = 0;
  if (TK == TK_RLE) {  // timestamp.rs:226-259
    uint64_t dl = 0;
    const bool ok = decode_varint(tpv.data + 10, tpv.data_len - 10, &dl);
    if (!ok) { if (lane == 0) report_error(P, TSKV_ERR_SHORT_BLOCK, tpage); return; }
    t_delta = dl * pow10_u64(__ldg(tpv.data + 1) & 0xf);
    t_first = load_be64_any(tpv.data + 2);
  } else {             // timestamp.rs:261-299
    const uint64_t scaler = pow10_u64(__ldg(tpv.data + 1) & 0xf);
    const uint32_t got = coop_decode_s8b<false>(tpv.data + 10, (tpv.data_len - 10) >> 3, load_be64_any(tpv.data + 2),
                                                scaler, S.ts, n_rows);
    if (got < n_rows) { if (lane == 0) report_error(P, TSKV_ERR_BITSET_MISMATCH, tpage); return; }
  }
  // ---- B. values + validity ranks -------------------------------------------------------------------
  const uint32_t *vbm = reinterpret_cast<const uint32_t *>(vpv.bitset);
  const uint32_t n_bm = (n_rows + 31) >> 5;
  uint32_t n_valid;
  {
    uint32_t w = 0;
    if (lane < n_bm) {
      w = __ldg(vbm + lane);
      if (lane == n_bm - 1 && (n_rows & 31)) w &= (1u << (n_rows & 31)) - 1;
    }
    const uint32_t ex = warp_excl_scan_u32(__popc(w), &n_valid);
    S.rank_base[lane] = ex;
  }
  if (VK == VK_S8B) {
    const uint32_t got = coop_decode_s8b<true>(vpv.data + 10, (vpv.data_len - 10) >> 3,
                                               (uint64_t)zigzag_dec(load_be64_any(vpv.data + 2)), 1, S.vals, n_valid);
    if (got < n_valid) { if (lane == 0) report_error(P, TSKV_ERR_BITSET_MISMATCH, page); return; }
  } else if (n_valid) {  // gorilla, phase 2: value i = first ^ xor of the elements' deltas 1..i
    const GorGroup &G = *reinterpret_cast<const GorGroup *>(&S.gor);
    const uint32_t n_parsed = G.n_parsed[g];  // < n_valid: element n_parsed + 1 ran past the block
    const uint32_t *wp;
    uint32_t base_bits, total_bits;
    gor_stream(vpv, wp, base_bits, total_bits);
    uint64_t carry = load_be64_any(vpv.data + 2);
    uint32_t first_sentinel = 0xffffffffu;  // lowest value index < n_valid (and before the overrun) holding the sentinel
    uint64_t v_end = 0;                     // value n_valid (has to be the sentinel)
    bool end_ok = false;
    // records were written by this kernel (phase 1): read them from L2, not through the read-only path. The loop is
    // software-pipelined: the record of tile t+2 and the window bits of tile t+1 are in flight during tile t's scan
    // (raw words of tile t+1 are loaded during tile t and only byte-swapped / shifted one iteration later)
    uint32_t rec_cur = (lane >= 1 && lane <= n_parsed) ? __ldcg(records + lane) : 0u;
    uint32_t rec_next = (lane + 32 <= n_parsed) ? __ldcg(records + lane + 32) : 0u;
    uint32_t w0 = 0, w1 = 0, w2 = 0;
    {
      const uint32_t wi = (base_bits + (rec_cur & 0x1ffff)) >> 5;
      if (rec_cur) { w0 = __ldg(wp + wi); w1 = __ldg(wp + wi + 1); w2 = __ldg(wp + wi + 2); }
    }
    for (uint32_t i0 = 0; i0 <= n_parsed; i0 += 32) {
      const uint32_t i = i0 + lane;
      // issue the next tile's loads first
      const uint32_t rec_n1 = rec_next;
      rec_next = (i + 64 <= n_parsed) ? __ldcg(records + i + 64) : 0u;
      uint32_t n0 = 0, n1 = 0, n2 = 0;
      {
        const uint32_t wi = (base_bits + (rec_n1 & 0x1ffff)) >> 5;
        if (rec_n1) { n0 = __ldg(wp + wi); n1 = __ldg(wp + wi + 1); n2 = __ldg(wp + wi + 2); }
      }
      // this tile: window bits -> delta (sig == 0: the first value or a "repeat" element, pushed without a sentinel test)
      const uint32_t sig = (rec_cur >> 17) & 0x7f;
      uint64_t delta = 0;
      if (sig) {
        const uint32_t sh = (base_bits + (rec_cur & 0x1ffff)) & 31;
        const uint32_t a = __byte_perm(w0, 0, 0x0123), b = __byte_perm(w1, 0, 0x0123), cc = __byte_perm(w2, 0, 0x0123);
        const uint64_t win = ((uint64_t)__funnelshift_l(b, a, sh) << 32) | __funnelshift_l(cc, b, sh);
        delta = (win >> (64 - sig)) << (rec_cur >> 24);
      }
      const uint64_t x = warp_incl_xor_scan_u64(delta) ^ carry;
      if (i < n_valid && i <= n_parsed) S.vals[cpad(i)] = x;
      const bool is_end = sig != 0 && x == GOR_SENTINEL;  // float.rs:585-589
      const uint32_t sm = __ballot_sync(FULL, i < n_valid && is_end);
      if (sm && first_sentinel == 0xffffffffu) first_sentinel = i0 + __ffs(sm) - 1;
      if (n_valid - i0 < 32 && n_parsed == n_valid) {
        v_end = shfl_u64(x, n_valid - i0);
        end_ok = __shfl_sync(FULL, (int)is_end, n_valid - i0) != 0;
      }
      carry = shfl_u64(x, 31);
      rec_cur = rec_n1; w0 = n0; w1 = n1; w2 = n2;
    }
    // the serial cursor's outcomes (cursors.cuh GorillaCursor): a sentinel before the bitset is served =
    // "Mismatch between bit set and decoded values"; running past the block = "unexpected end of block"
    if (first_sentinel != 0xffffffffu) { if (lane == 0) report_error(P, TSKV_ERR_BITSET_MISMATCH, page); return; }
    if (n_parsed < n_valid) { if (lane == 0) report_error(P, TSKV_ERR_SHORT_BLOCK, page); return; }
    if (!end_ok) {
      // more elements than valid rows: the reference decodes on to the sentinel (float.rs:480-591). Rare; every
      // lane walks the rest of the stream redundantly.
      uint32_t bitpos = G.endpos[g], meaningful = G.meaningful[g], trailing = G.trailing[g];
      uint64_t val = v_end;
      for (;;) {
        uint32_t sig;
        const uint32_t len = gor_parse_ctrl(gor_peek32(wp, base_bits + bitpos) >> 19, meaningful, trailing, sig);
        if (sig) val ^= (gor_peek64(wp, base_bits + bitpos + len) >> (64 - sig)) << (trailing & 63);
        bitpos += len + sig;
        if (bitpos > total_bits) { if (lane == 0) report_error(P, TSKV_ERR_SHORT_BLOCK, page); return; }
        if (sig && val == GOR_SENTINEL) break;
      }
    }
  }
  __syncwarp();
  // ---- C. per-row keys -> segment heads ---------------------------------------------------------------
  bool range_err = false;
  uint32_t n_seg = 0, n_inrange = 0;
  uint32_t prev_key = 0xfffffffeu;  // key of the row before this 32-row strip (lane 31 of the last strip)
  for (uint32_t r0 = 0; r0 < n_rows; r0 += 32) {
    const uint32_t r = r0 + lane;
    uint32_t key = 0xfffffffeu;
    if (r < n_rows) {
      const int64_t t = TK == TK_RLE ? (int64_t)(t_first + (uint64_t)r * t_delta) : (int64_t)S.ts[cpad(r)];
      key = coop_row_key(P, C, t, &range_err);
    }
    uint32_t left = __shfl_up_sync(FULL, key, 1);
    if (lane == 0) left = prev_key;
    const bool head = r < n_rows && key != left;
    const uint32_t hm = __ballot_sync(FULL, head);
    if (head) S.seg[n_seg + __popc(hm & ((1u << lane) - 1))] = (uint16_t)r;
    n_seg += __popc(hm);
    n_inrange += __popc(__ballot_sync(FULL, r < n_rows && key != 0xffffffffu));
    prev_key = __shfl_sync(FULL, key, 31);
  }
  if (lane == 0) S.seg[n_seg] = (uint16_t)n_rows;
  __syncwarp();
  if (__any_sync(FULL, range_err)) {
    if (lane == 0) report_error(P, TSKV_ERR_BUCKET_RANGE, page);
    return;
  }
  // ---- D. lane-per-segment reduce ---------------------------------------------------------------------
  const uint64_t flip = pt == TSKV_PT_U64 ? 0x8000000000000000ull : 0ull;
  const bool mean_hi = (mask & TSKV_AGG_MEAN) != 0;
  const uint64_t group_base = group_cell_base(P, slot);
  for (uint32_t s0 = 0; s0 < n_seg; s0 += 32) {
    const uint32_t s = s0 + lane;
    if (s < n_seg) {
      const uint32_t rb = S.seg[s], re = S.seg[s + 1];
      const int64_t tb = TK == TK_RLE ? (int64_t)(t_first + (uint64_t)rb * t_delta) : (int64_t)S.ts[cpad(rb)];
      bool dummy = false;
      const uint32_t key = coop_row_key(P, C, tb, &dummy);
      if (key != 0xffffffffu) {
        ValueAcc<VK> va;
        va.reset();
        uint64_t first_v = 0, last_v = 0;
        bool first_ok = false, last_ok = false;
        for (uint32_t r = rb; r < re; r++) {
          const uint32_t w = __ldg(vbm + (r >> 5));
          const bool vv = (w >> (r & 31)) & 1;
          uint64_t v = 0;
          if (vv) {
            v = S.vals[cpad(S.rank_base[r >> 5] + __popc(w & ((1u << (r & 31)) - 1)))];
            va.count++;
            va.add(v, pt, flip, mean_hi);
          }
          if (SEL) {
            if (r == rb) { first_v = v; first_ok = vv; }
            last_v = v;
            last_ok = vv;
          }
        }
        const uint64_t cell = group_base + key;
        va.fold(pt);
        if (va.count) table_update(P, stab, cs, cell, mask, VK == VK_GOR, va.count, va.sum, va.sum_hi, va.kmin, va.kmax);
        if (SEL) {
          const int64_t te = TK == TK_RLE ? (int64_t)(t_first + (uint64_t)(re - 1) * t_delta) : (int64_t)S.ts[cpad(re - 1)];
          int64_t kf = tb, kl = te;
          if (P.slot_bits) {
            const uint64_t kb = P.width > 0 ? (uint64_t)P.first_bucket_start + (uint64_t)((int64_t)key - 1) * (uint64_t)P.width
                                            : (uint64_t)P.rel_base;
            kf = (int64_t)((((uint64_t)tb - kb) << P.slot_bits) | slot);
            kl = (int64_t)((((uint64_t)te - kb) << P.slot_bits) | (P.slot_max - slot));
          }
          if ((mask & TSKV_AGG_FIRST) && first_ok) atomic_select_pair<true>(P.state + cs.first_off + 2 * cell, kf, first_v);
          if ((mask & TSKV_AGG_LAST) && last_ok) atomic_select_pair<false>(P.state + cs.last_off + 2 * cell, kl, last_v);
        }
      }
    }
  }
  __syncwarp();
  if (lane == 0) {
    atomicAdd(&P.stats[0], (unsigned long long)n_valid);
    if (n_inrange) atomicAdd(&P.stats[1], (unsigned long long)n_inrange);
  }
}

template <int TK, int VK, bool SEL>
__global__ void __launch_bounds__(SCAN_THREADS, 2) k_scan_coop(const __grid_constant__ ScanParams P,
                                                               const __grid_constant__ CoopParams C, int bin) {
  extern __shared__ __align__(16) uint64_t s_dyn[];  // [per-CTA table | per-warp CoopSmem]
  uint64_t *s_tab = s_dyn;
  if (P.use_smem) {
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
  using Smem = CoopSmem<TK == TK_S8B, VK == VK_GOR>;
  Smem &S = *reinterpret_cast<Smem *>(reinterpret_cast<uint8_t *>(s_dyn + ((P.smem_words + 1) & ~1u)) +
                                      (threadIdx.x >> 5) * ((sizeof(Smem) + 15) & ~(size_t)15));
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t begin0 = __ldg(P.bin_cstart + bin), end0 = __ldg(P.bin_cstart + bin + 1);
  if (VK != VK_GOR) {
    for (;;) {
      uint32_t i = 0;
      if (lane == 0) i = atomicAdd(P.task_counter + bin, 1u);
      i = __shfl_sync(FULL, i, 0);
      if (begin0 + i >= end0) break;
      scan_page_coop<TK, VK, SEL>(P, C, begin0 + i, S, s_tab);
      __syncwarp();
    }
  } else {
    const uint32_t group = C.gor_group;
    uint32_t *rows = C.gor_scratch[bin == BIN_COOP_RLE_GOR ? 0 : 1] +
                     (size_t)(blockIdx.x * (SCAN_THREADS / 32) + (threadIdx.x >> 5)) * group * GOR_REC_STRIDE;
    GorGroup &G = *reinterpret_cast<GorGroup *>(&S.gor);
    for (;;) {
      uint32_t t = 0;
      if (lane == 0) t = atomicAdd(P.task_counter + bin, 1u);
      t = __shfl_sync(FULL, t, 0);
      const uint64_t first = (uint64_t)begin0 + (uint64_t)t * group;
      if (first >= end0) break;
      const uint32_t cnt = min(group, end0 - (uint32_t)first);
      // phase 1
      if (group == 1) gor_parse_page_staged(P, (uint32_t)first, rows, G, reinterpret_cast<uint32_t *>(&S), (uint32_t)(offsetof(Smem, gor) / 4));
      else if (lane < cnt) gor_parse_page(P, (uint32_t)first + lane, rows + lane * GOR_REC_STRIDE, G, lane);
      __syncwarp();
      for (uint32_t g = 0; g < cnt; g++) {                                                            // phase 2
        scan_page_coop<TK, VK, SEL>(P, C, (uint32_t)first + g, S, s_tab, rows + g * GOR_REC_STRIDE, g);
        __syncwarp();
      }
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

}  // namespace tskv
