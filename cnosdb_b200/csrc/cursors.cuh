// cursors.cuh — per-lane streaming decoders for TSM column pages (sm_90a).
//
// Design: one lane owns one page and walks it value by value, so decode -> filter -> bucket
// reduce happens in registers and no decoded value is ever written to HBM. The formats are those of
// the reference codecs (all paths relative to the reference tree):
//   page framing     tskv/src/tsm/page.rs:31-94
//   simple8b         tskv/src/tsm/codec/simple8b.rs:80-208
//   timestamp delta  tskv/src/tsm/codec/timestamp.rs:177-299   (deltas NOT zig-zagged, 10^k scaler)
//   integer delta    tskv/src/tsm/codec/integer.rs:142-248     (zig-zag deltas)
//   gorilla          tskv/src/tsm/codec/float.rs:418-606
//   raw ("Null")     tskv/src/tsm/codec/timestamp.rs:301-323, float.rs:387-413
// Arithmetic wraps like the reference's release build (Cargo.toml:190-197).
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#include "../../include/tskv_gpu.h"
#include "kinds.h"

namespace tskv {

// Bytes allocated (and zeroed) after the last page of a device arena: streaming loads read whole aligned words /
// 16-byte chunks and may run past the end of the last page (compute-sanitizer memcheck, round 2: the 64 bytes of
// round 1 were less than its 72-byte look-ahead).
constexpr uint32_t ARENA_SLACK = 256;

__device__ __forceinline__ uint64_t bswap64(uint64_t v) {
  uint32_t lo = (uint32_t)v, hi = (uint32_t)(v >> 32);
  return ((uint64_t)__byte_perm(lo, 0, 0x0123) << 32) | __byte_perm(hi, 0, 0x0123);
}
__device__ __forceinline__ int64_t zigzag_dec(uint64_t v) {
  return (int64_t)((v >> 1) ^ (0 - (v & 1)));
}

// Streams an arbitrarily aligned byte range as big-endian u64 words. Two implementations with the
// same interface:
//   BeStream      aligned 8-byte global loads (one per word; previous word kept and funnel-shifted). Reads up to
//                 15 bytes past the end of the range (the arena carries ARENA_SLACK bytes after the last page).
//   SeqStream     the same words staged through a per-lane shared-memory ring of 16-byte cp.async chunks (below).
struct BeStream {
  const uint64_t *ap;  // next aligned word
  uint64_t cur;        // last aligned word, little-endian
  uint32_t sh;         // misalignment in bits
  __device__ __forceinline__ void init(const uint8_t *p, uint32_t /*smem_slot*/ = 0, const uint8_t * /*end*/ = nullptr) {
    uintptr_t a = reinterpret_cast<uintptr_t>(p);
    sh = (uint32_t)(a & 7) * 8;
    ap = reinterpret_cast<const uint64_t *>(a & ~(uintptr_t)7);
    cur = __ldg(ap++);
  }
  __device__ __forceinline__ void reset(uint32_t /*lane_slot*/ = 0) {}
  __device__ __forceinline__ uint64_t next() {
    uint64_t nxt = __ldg(ap++);
    uint64_t raw = (cur >> sh) | ((nxt << 1) << (63 - sh));
    cur = nxt;
    return bswap64(raw);
  }
};

// ------------------------------------------------------------------------------------------------
// Shared-memory staging of a lane's byte stream (round 2). One lane owns one page, so a warp reads 32 different
// pages: each lane stages ITS stream through a private ring of RING_CHUNKS 16-byte chunks filled by 128-bit cp.async
// (LDGSTS.128, L2 -> shared memory without a register round trip). A lane's ring is contiguous (RING_BYTES bytes) and
// the lanes' rings are RING_BYTES apart. Each lane's chunk slots are rotated by its lane index: chunk c of the stream
// lives at slot (c + rot) mod RING_CHUNKS, rot = lane mod RING_CHUNKS. Without the rotation every ring would start on
// the same bank; with it, lanes that sit at the same stream offset spread over min(RING_CHUNKS, 8) 16-byte bank groups,
// as a 16-byte skew between the rings would, without the skew's 16 bytes per lane. The rotation costs nothing per word:
// the decoders keep their stream positions in RING COORDINATES, i.e. counted from chunk rot (word index k = the word's
// index from the stream's aligned start + 2 rot, bit position + 128 rot), so word k lives at
//   ring + lane * RING_BYTES + (k mod 2 * RING_CHUNKS) * 8
// (one AND + one scaled add per word). Restart points (SkipEntry) hold positions relative to the stream's start, so an
// entry saved by one lane restores on any other.
// A decoder calls step(c) once per element / word BEFORE reading, c = the chunk its read window starts in; a window
// never spans more than chunks c and c + 1, and c advances by at most one per step (an element is <= 77 bits, a word
// 64). step() issues at most one new chunk - a predicated LDGSTS - commits exactly one group and waits until at most
// RING_CHUNKS - 2 groups are pending: chunk c + 1 was issued when the window first reached chunk c + 2 - RING_CHUNKS,
// i.e. at least RING_CHUNKS - 2 steps (= groups) ago, so it has landed; the RING_CHUNKS - 2 chunks behind it (96
// bytes, ~12 full-mantissa gorilla values) stay in flight and hide the HBM / L2 latency.
// The initial fill is one group the caller waits for once per page (ring_drain) before the first step.
// A stream is read at most RING_BYTES + 15 bytes past its last byte (the initial fill of a short stream; otherwise up to
// the end of its last 16-byte chunk): the following pages, or the ARENA_SLACK bytes after the last page of the arena -
// never past the allocation. A decoder that consumes bytes past its block reads stale shared memory, and its own
// end-of-stream accounting reports the overrun.
#ifndef TSKV_RING_CHUNKS
#define TSKV_RING_CHUNKS 8
#endif
constexpr int RING_CHUNKS = TSKV_RING_CHUNKS;
constexpr uint32_t RING_BYTES = RING_CHUNKS * 16;       // one lane, one stream
constexpr uint32_t RING_BYTES_PER_WARP = 32 * RING_BYTES;  // one stream of one warp
static_assert((RING_CHUNKS & (RING_CHUNKS - 1)) == 0 && RING_CHUNKS >= 4, "ring size must be a power of two >= 4");
static_assert(ARENA_SLACK >= RING_BYTES + 32, "the arena slack has to cover the rings' read-ahead");

struct ChunkRing {
  const uint8_t *gnext;  // global address of the next chunk to issue (16-byte aligned)
  uint32_t sbase;        // shared-space address of this lane's ring
  uint32_t snext;        // ring offset (bytes) the next chunk goes to
  uint32_t trig;         // the next chunk is issued once the read window reaches chunk `trig` (0xffffffff: none left)
  uint32_t trig_last;    // value of `trig` at which the page's last chunk goes out
  // The calling lane's rotation in chunks (ring coordinates, above). The ring always belongs to the calling lane, so
  // the rotation comes from the lane index rather than from per-ring state.
  static __device__ __forceinline__ uint32_t rot() { return threadIdx.x & 31 & (RING_CHUNKS - 1); }
  __device__ __forceinline__ void issue_one() {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" :: "r"(sbase + snext), "l"(gnext) : "memory");
    gnext += 16;
    snext = (snext + 16) & (RING_BYTES - 1);
  }
  __device__ __forceinline__ void init(const uint8_t *start, const uint8_t *end, uint32_t lane_ring) {
    const uintptr_t a = reinterpret_cast<uintptr_t>(start) & ~(uintptr_t)15, e = reinterpret_cast<uintptr_t>(end);
    const uint32_t r = rot();
    gnext = reinterpret_cast<const uint8_t *>(a);
    const uint32_t n_chunks = e > a ? (uint32_t)((e - a + 15) >> 4) : 0u;  // chunks that intersect the stream
    sbase = lane_ring;
    snext = r * 16;  // the stream's first chunk
#pragma unroll
    for (int i = 0; i < RING_CHUNKS; i++) issue_one();  // (a short stream's fill reads < RING_BYTES past its end)
    trig = n_chunks > RING_CHUNKS ? r + 1 : 0xffffffffu;  // chunk RING_CHUNKS goes out when the window reaches chunk 1
    trig_last = n_chunks - RING_CHUNKS + r;
  }
  // The same ring entered in the middle of the stream (restart points, SkipEntry below): the first chunk staged is
  // chunk c0, in ring coordinates like every chunk / word index of the decoders.
  __device__ __forceinline__ void init_at(const uint8_t *start, const uint8_t *end, uint32_t lane_ring, uint32_t c0) {
    const uintptr_t a = reinterpret_cast<uintptr_t>(start) & ~(uintptr_t)15, e = reinterpret_cast<uintptr_t>(end);
    const uint32_t r = rot();
    const uint32_t n_chunks = e > a ? (uint32_t)((e - a + 15) >> 4) : 0u;
    gnext = reinterpret_cast<const uint8_t *>(a) + (size_t)(c0 - r) * 16;
    sbase = lane_ring;
    snext = (c0 & (RING_CHUNKS - 1)) * 16;
#pragma unroll
    for (int i = 0; i < RING_CHUNKS; i++) issue_one();  // (near the end of the stream: < RING_BYTES past its end)
    trig = n_chunks + r > c0 + RING_CHUNKS ? c0 + 1 : 0xffffffffu;
    trig_last = n_chunks - RING_CHUNKS + r;
  }
  // One decoder step whose read window starts in chunk c (see above). Nothing is issued past the stream's last chunk,
  // however far a decoder that ran off a truncated block pushes its window.
  __device__ __forceinline__ void step(uint32_t c) {
    if (c >= trig) {
      issue_one();
      trig = trig == trig_last ? 0xffffffffu : trig + 1;
    }
    asm volatile("cp.async.commit_group;\n\tcp.async.wait_group %0;\n" :: "n"(RING_CHUNKS - 2) : "memory");
  }
  // An idle ring: steps issue nothing (lanes without a page / kinds without a stream).
  __device__ __forceinline__ void reset(uint32_t lane_ring) { gnext = nullptr; sbase = lane_ring; snext = 0; trig = 0xffffffffu; trig_last = 0; }
  static __device__ __forceinline__ uint2 lds64(uint32_t addr) {
    uint2 v;
    asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];\n" : "=r"(v.x), "=r"(v.y) : "r"(addr) : "memory");
    return v;
  }
  // 64-bit word k of the stream (8-byte units, ring coordinates), as stored (little-endian load of stream bytes)
  __device__ __forceinline__ uint2 word(uint32_t k) const { return lds64(sbase + ((k & (2 * RING_CHUNKS - 1)) << 3)); }
  // words k, k + 1, k + 2
  __device__ __forceinline__ void words3(uint32_t k, uint2 &w0, uint2 &w1, uint2 &w2) const {
    w0 = word(k);
    w1 = word(k + 1);
    w2 = word(k + 2);
  }
};
// Commits the initial fills of the lane's rings and waits for them (once per page, before the first step).
__device__ __forceinline__ void ring_drain() { asm volatile("cp.async.commit_group;\n\tcp.async.wait_all;\n" ::: "memory"); }

// ------------------------------------------------------------------------------------------------
// Restart points (round 2, "skip index"). A page is one serial stream: the value of row r depends on every element
// before it, so one page is one dependent chain of ~1000 elements however many SMs are idle. TSM pages are immutable,
// so the page set carries - built ONCE, on the device, when the pages are uploaded (k_build_skip) - the decoder state
// at every SKIP_ROWS-th row of every simple8b / gorilla page: 16 bytes per restart point. A scan then cuts a page into
// parts of m * SKIP_ROWS rows, each decoded by its own lane from the restart point (RLE pages need none: closed form).
// The entry is the cursor's own state (save() / restore() below), so a restarted cursor continues bit-identically:
//   simple8b (S8bCursor):  v = running value, a = aligned-word index of the stream position (relative to the
//                          stream's first word), b = values left in the current packed word
//   gorilla (GorillaRing): v = the value the next call returns, a = bit position of the following element (relative
//                          to the stream's first bit), b = meaningful | trailing << 8 | cur_ok << 16 | any << 17
// ------------------------------------------------------------------------------------------------
#ifndef TSKV_SKIP_ROWS
#define TSKV_SKIP_ROWS 128
#endif
constexpr uint32_t SKIP_ROWS = TSKV_SKIP_ROWS;  // a multiple of 32 (bitmap words)
static_assert(SKIP_ROWS % 32 == 0 && SKIP_ROWS >= 32, "restart points sit on bitmap-word boundaries");
constexpr uint32_t SKIP_NONE = 0xffffffffu;
struct SkipEntry {
  uint64_t v;
  uint32_t a, b;
};
static_assert(sizeof(SkipEntry) == 16, "restart points are 16-byte records");
__device__ __forceinline__ SkipEntry load_skip(const SkipEntry *p) {
  const uint4 r = __ldg(reinterpret_cast<const uint4 *>(p));
  SkipEntry e;
  e.v = ((uint64_t)r.y << 32) | r.x;
  e.a = r.z;
  e.b = r.w;
  return e;
}

// Sequential big-endian u64 words of an arbitrarily aligned byte range through a ChunkRing (simple8b / raw pages).
// Same interface as BeStream.
struct SeqStream {
  ChunkRing ring;
  uint32_t k;     // index of the last aligned word loaded (ring coordinates)
  uint32_t psel;  // byte-permute selector: the big-endian word at the stream's (constant) byte misalignment
  bool high;      // the misalignment is >= 4 bytes
  uint2 cur;      // last aligned word, as stored
  __device__ __forceinline__ void init(const uint8_t *p, uint32_t lane_slot, const uint8_t *end) {
    ring.init(p, end, lane_slot);
    const uintptr_t a = reinterpret_cast<uintptr_t>(p);
    const uint32_t o = (uint32_t)(a & 7), q = o & 3;
    high = o >= 4;
    psel = (q + 3) | ((q + 2) << 4) | ((q + 1) << 8) | (q << 12);  // result byte 3 (most significant) = stream byte q
    k = first_word_index(p);
    const uint64_t w = __ldg(reinterpret_cast<const uint64_t *>(a & ~(uintptr_t)7));  // the first word straight from global memory
    cur = make_uint2((uint32_t)w, (uint32_t)(w >> 32));
  }
  // Enters the stream at aligned word k0 + rel (k0 = the index init() starts at): the next next() composes the packed
  // word that starts in aligned word k0 + rel.
  __device__ __forceinline__ void init_at(const uint8_t *p, uint32_t lane_slot, const uint8_t *end, uint32_t rel) {
    const uintptr_t a = reinterpret_cast<uintptr_t>(p);
    const uint32_t o = (uint32_t)(a & 7), q = o & 3;
    high = o >= 4;
    psel = (q + 3) | ((q + 2) << 4) | ((q + 1) << 8) | (q << 12);
    const uint32_t kk = ((uint32_t)(a & 15) >> 3) + rel;  // from the aligned start
    k = kk + 2 * ChunkRing::rot();
    ring.init_at(p, end, lane_slot, k >> 1);
    const uint64_t w = __ldg(reinterpret_cast<const uint64_t *>(a & ~(uintptr_t)15) + kk);
    cur = make_uint2((uint32_t)w, (uint32_t)(w >> 32));
  }
  // ring-coordinate index of the aligned word that holds the stream's first byte
  static __device__ __forceinline__ uint32_t first_word_index(const uint8_t *p) {
    return ((uint32_t)(reinterpret_cast<uintptr_t>(p) & 15) >> 3) + 2 * ChunkRing::rot();
  }
  __device__ __forceinline__ uint64_t next() {
    k++;
    ring.step(k >> 1);
    const uint2 nxt = ring.word(k);
    // bytes o .. o + 7 of (cur, nxt), most significant first: two byte permutes over three of the four 32-bit words
    const uint32_t a = high ? cur.y : cur.x, b = high ? nxt.x : cur.y, c = high ? nxt.y : nxt.x;
    const uint32_t hi = __byte_perm(a, b, psel), lo = __byte_perm(b, c, psel);
    cur = nxt;
    return ((uint64_t)hi << 32) | lo;
  }
  __device__ __forceinline__ void reset(uint32_t lane_slot = 0) { ring.reset(lane_slot); k = 0; psel = 0x0123; high = false; cur = make_uint2(0, 0); }
};

__device__ __forceinline__ uint64_t load_be64(const uint8_t *p) {
  BeStream s;
  s.init(p);
  return s.next();
}
__device__ __forceinline__ uint32_t load_be32_aligned(const uint8_t *p) {
  return __byte_perm(__ldg(reinterpret_cast<const uint32_t *>(p)), 0, 0x0123);
}

// Parsed page header (page.rs:78-94).
struct PageView {
  const uint8_t *bitset;  // 16-byte aligned (page offset is)
  const uint8_t *data;
  uint32_t data_len;
  uint32_t n_rows;
  __device__ __forceinline__ void open(const uint8_t *arena, const tskv_page_desc &d) {
    const uint8_t *pg = arena + d.offset;
    uint4 h = __ldg(reinterpret_cast<const uint4 *>(pg));
    uint32_t bitset_len = __byte_perm(h.x, 0, 0x0123);
    // rows: u64 BE at [4..12); the host validated it equals desc.num_values (< 2^32)
    n_rows = d.num_values;
    bitset = pg + 16;
    data = pg + 16 + bitset_len;
    data_len = d.size - 16 - bitset_len;
  }
};

// Validity bitmap, Arrow LSB-first (page.rs:78-84).
struct BitCursor {
  const uint32_t *wp;
  uint32_t word, ahead;  // `ahead` = the next 32 rows, loaded one word early to hide the latency
  __device__ __forceinline__ void init(const uint8_t *bitset) {
    wp = reinterpret_cast<const uint32_t *>(bitset);
    word = 0;
    ahead = __ldg(wp++);
  }
  // `row` must advance by one per call starting at 0. Reads at most 8 bytes past the bitmap.
  __device__ __forceinline__ bool next(uint32_t row) {
    if ((row & 31) == 0) {
      word = ahead;
      ahead = __ldg(wp++);
    }
    bool b = word & 1;
    word >>= 1;
    return b;
  }
};

__constant__ uint8_t c_s8b_count[16] = {240, 120, 60, 30, 20, 15, 12, 10, 8, 7, 6, 5, 4, 3, 2, 1};
__constant__ uint8_t c_s8b_bits[16] = {0, 0, 1, 2, 3, 4, 5, 6, 7, 8, 10, 12, 15, 20, 30, 60};
// The same tables (simple8b.rs:17-50) as byte-permute lookups: lanes of a warp decode different pages and hold
// different selectors, and a divergent index into constant memory is replayed once per distinct value.
__device__ __forceinline__ void s8b_lut(uint32_t sel, uint32_t &count, uint32_t &bits) {
  const uint32_t i = sel & 7;
  const uint32_t c_lo = __byte_perm(0x1e3c78f0u, 0x0a0c0f14u, i);  // 240 120 60 30 | 20 15 12 10
  const uint32_t c_hi = __byte_perm(0x05060708u, 0x01020304u, i);  //   8   7  6  5 |  4  3  2  1
  const uint32_t b_lo = __byte_perm(0x02010000u, 0x06050403u, i);  //   0   0  1  2 |  3  4  5  6
  const uint32_t b_hi = __byte_perm(0x0c0a0807u, 0x3c1e140fu, i);  //   7   8 10 12 | 15 20 30 60
  const bool hi = sel & 8;
  count = (hi ? c_hi : c_lo) & 0xff;
  bits = (hi ? b_hi : b_lo) & 0xff;
}

// LEB128 (integer-encoding 4.0.2 decode_var); returns false when the slice ends first.
__device__ inline bool decode_varint(const uint8_t *p, uint32_t len, uint64_t *out) {
  uint64_t r = 0;
  uint32_t shift = 0;
  for (uint32_t i = 0; i < len; i++) {
    uint8_t b = __ldg(p + i);
    if (shift < 64) r |= (uint64_t)(b & 0x7f) << shift;
    shift += 7;
    if ((b & 0x80) == 0) {
      *out = r;
      return true;
    }
    if (shift > 63) return false;
  }
  return false;
}

__device__ __forceinline__ uint64_t pow10_u64(uint32_t k) {
  uint64_t s = 1;
  for (uint32_t i = 0; i < k; i++) s *= 10;
  return s;
}

// ------------------------------------------------------------------------------------------------
// Delta-family cursor: RLE / simple8b / raw prefix sum / raw BE, zig-zag or scaled.
// KIND is one of the DK_* delta kinds, or -1 for a runtime switch on `kind` (generic path).
// next() has no "first value" special case: open() arranges the state so that the first call
// yields the page's first value (RLE: v = first - delta; simple8b: one fake zero delta queued).
// Running out of encoded values sets the sticky `exhausted` flag (and yields garbage): callers check
// it once per segment / page instead of once per value.
// ------------------------------------------------------------------------------------------------
template <int KIND, typename STREAM = BeStream>
struct DeltaCursor {
  STREAM bs;
  uint64_t v;           // running value (raw bits)
  uint64_t delta;       // RLE delta (already scaled / zig-zag decoded)
  uint64_t scaler;      // S8B_SC
  uint64_t w;           // current simple8b word, consumed from the low bits
  uint64_t mask;        // low `bits` bits
  uint32_t words_left;  // 8-byte words not yet loaded
  uint32_t in_word;     // values left in `w`
  uint32_t bits;        // width of one value in `w`
  uint32_t ones;        // 1 for the run-of-ones selectors (payload ignored), else 0
  uint8_t kind;         // runtime kind (== KIND when KIND >= 0)
  bool exhausted;

  __device__ __forceinline__ int k() const { return KIND >= 0 ? KIND : kind; }

  // Returns TSKV_OK or a decode error. `pv.data` starts at the Encoding id byte; the host already
  // classified the page, so lengths needed by the fixed header are guaranteed.
  __device__ inline tskv_status open(const PageView &pv, uint8_t kind_, uint32_t smem_slot = 0) {
    kind = KIND >= 0 ? (uint8_t)KIND : kind_;
    bs.reset(smem_slot);
    exhausted = false;
    v = 0;
    delta = 0;
    scaler = 1;
    w = 0;
    mask = 0;
    in_word = 0;
    bits = 0;
    ones = 0;
    words_left = 0;
    const uint8_t *d = pv.data;
    switch (k()) {
      case DK_RLE_SC: {  // timestamp.rs:226-259: data = id | kind/scaler | first(8) | varint delta | varint n
        uint64_t dl;
        if (!decode_varint(d + 10, pv.data_len - 10, &dl)) return TSKV_ERR_SHORT_BLOCK;
        delta = dl * pow10_u64(__ldg(d + 1) & 0xf);
        v = load_be64(d + 2) - delta;
        break;
      }
      case DK_RLE_ZZ: {  // integer.rs:186-214
        uint64_t dl;
        if (!decode_varint(d + 10, pv.data_len - 10, &dl)) return TSKV_ERR_SHORT_BLOCK;
        delta = (uint64_t)zigzag_dec(dl);
        v = (uint64_t)zigzag_dec(load_be64(d + 2)) - delta;
        break;
      }
      case DK_S8B_SC:  // timestamp.rs:261-299
        scaler = pow10_u64(__ldg(d + 1) & 0xf);
        v = load_be64(d + 2);  // header fields come straight from global memory; the stream covers the packed words
        bs.init(d + 10, smem_slot, d + pv.data_len);
        words_left = (pv.data_len - 10) >> 3;
        in_word = 1;  // fake zero delta in front of the packed ones
        break;
      case DK_S8B_ZZ:  // integer.rs:216-248
        v = (uint64_t)zigzag_dec(load_be64(d + 2));
        bs.init(d + 10, smem_slot, d + pv.data_len);
        words_left = (pv.data_len - 10) >> 3;
        in_word = 1;
        break;
      case DK_RAW_SC:  // timestamp.rs:201-224
      case DK_RAW_ZZ:  // integer.rs:165-184
        bs.init(d + 2, smem_slot, d + pv.data_len);
        words_left = (pv.data_len - 2) >> 3;
        break;
      case DK_RAWBE:  // timestamp.rs:301-323
        bs.init(d + 1, smem_slot, d + pv.data_len);
        words_left = (pv.data_len - 1) >> 3;
        break;
      case DK_BOOL_PACK: {  // boolean.rs:79-111: id | 0x10 | varint count | bits, MSB first
        uint64_t count = 0;
        uint32_t vl = 0, shift = 0;
        for (;; vl++) {  // (the host checked that the varint ends inside the block)
          const uint8_t b = __ldg(d + 2 + vl);
          if (shift < 64) count |= (uint64_t)(b & 0x7f) << shift;
          shift += 7;
          if (!(b & 0x80)) break;
        }
        vl++;
        const uint64_t have = (uint64_t)(pv.data_len - 2 - vl) * 8;  // bits the block really holds (src[bit_index / 8])
        words_left = (uint32_t)min(min(count, have), (uint64_t)0xffffffffu);   // VALUES left
        bs.init(d + 2 + vl, smem_slot, d + pv.data_len);
        break;
      }
      case DK_BOOL_RAW:  // boolean.rs:112-140: id | one byte per value
        words_left = pv.data_len - 1;  // VALUES left
        bs.init(d + 1, smem_slot, d + pv.data_len);
        break;
      default:
        break;
    }
    return TSKV_OK;
  }
  // Next boolean: `w` holds the unread part of the current 64-bit chunk of the stream, MSB first.
  __device__ __forceinline__ uint64_t next_bool(uint32_t width) {
    if (words_left == 0) {  // "Insufficient data for decoding" / the block ends before the bitset is served
      exhausted = true;
      return 0;
    }
    words_left--;
    if (in_word == 0) {
      w = bs.next();
      in_word = 64 / width;
    }
    in_word--;
    const uint64_t v = w >> (64 - width);
    w <<= width;
    return width == 1 ? v : (v == 1 ? 1ull : 0ull);
  }

  __device__ __forceinline__ void refill() {
    if (words_left == 0) {
      exhausted = true;
      in_word = 0x7fffffff;  // keep yielding zeros without refilling again
      w = 0; mask = 0; bits = 0; ones = 0;
      return;
    }
    words_left--;
    w = bs.next();
    const uint32_t sel = (uint32_t)(w >> 60);
    s8b_lut(sel, in_word, bits);
    ones = sel < 2 ? 1u : 0u;
    mask = bits ? (~0ull >> (64 - bits)) : 0ull;
  }
  // Next simple8b payload value (simple8b.rs:95-208).
  __device__ __forceinline__ uint64_t next_packed() {
    if (in_word == 0) refill();
    in_word--;
    const uint64_t u = (w & mask) | ones;
    w >>= bits;  // bits <= 60
    return u;
  }
  __device__ __forceinline__ uint64_t next_word() {
    if (words_left == 0) {
      exhausted = true;
      return 0;
    }
    words_left--;
    return bs.next();
  }

  // Value for the next VALID row.
  __device__ __forceinline__ uint64_t next() {
    switch (k()) {
      case DK_RLE_SC:
      case DK_RLE_ZZ: v += delta; return v;
      case DK_S8B_SC: v += next_packed() * scaler; return v;
      case DK_S8B_ZZ: v += (uint64_t)zigzag_dec(next_packed()); return v;
      case DK_RAW_SC: v += next_word(); return v;
      case DK_RAW_ZZ: v += (uint64_t)zigzag_dec(next_word()); return v;
      case DK_RAWBE: return next_word();
      case DK_BOOL_PACK: return next_bool(1);
      case DK_BOOL_RAW: return next_bool(8);
      default: exhausted = true; return 0;  // DK_ALLNULL never reaches here with a valid bit
    }
  }

  // timestamp.rs:273-279 quirk: with simple8b timestamps a NULL row 0 swallows the first value.
  __device__ __forceinline__ void skip_first_if_s8b_sc() {
    if (k() == DK_S8B_SC) in_word = 0;
  }
};

// ------------------------------------------------------------------------------------------------
// Lean simple8b delta cursor of the fused scan: DK_S8B_SC (ZZ = false: timestamps, deltas * 10^k, timestamp.rs:261-299)
// or DK_S8B_ZZ (ZZ = true: zig-zag deltas, integer.rs:216-248) through a staged SeqStream. Same values as
// DeltaCursor, less bookkeeping per word - the timestamp stream of an irregular series holds ONE 60-bit value per
// word, so per-word work is per-row work there:
//   * selector 15 (1 x 60 bits) takes a branch of its own (warp-uniform on such pages) instead of the table lookup;
//   * running out of words is not tracked per refill: the stream position says how many words were consumed, and
//     exhausted() compares it with the block's word count when the caller checks (after a segment). A cursor that ran
//     past its block decodes stale bytes in the meantime, which the caller discards with the error.
// ------------------------------------------------------------------------------------------------
template <bool ZZ>
struct S8bCursor {
  SeqStream bs;
  uint64_t v;        // running value (raw bits)
  uint64_t scaler;   // !ZZ
  uint64_t w;        // current word, consumed from the low bits
  uint64_t mask;     // low `bits` bits
  uint32_t in_word;  // values left in `w`
  uint32_t bits;
  uint32_t ones;     // 1 for the run-of-ones selectors (payload ignored)
  uint32_t k_end;    // stream word index of the block's last word

  __device__ __forceinline__ tskv_status open(const PageView &pv, uint8_t /*kind*/, uint32_t lane_ring) {
    const uint8_t *d = pv.data;
    scaler = ZZ ? 1 : pow10_u64(__ldg(d + 1) & 0xf);
    const uint64_t first = load_be64(d + 2);  // header fields straight from global memory; the stream covers the packed words
    v = ZZ ? (uint64_t)zigzag_dec(first) : first;
    bs.init(d + 10, lane_ring, d + pv.data_len);
    k_end = bs.k + ((pv.data_len - 10) >> 3);
    w = 0; mask = 0; bits = 0; ones = 0;
    in_word = 1;  // a fake zero delta in front of the packed ones: the first next() yields the first value
    return TSKV_OK;
  }
  __device__ __forceinline__ void reset(uint32_t lane_ring) {
    bs.reset(lane_ring);
    v = 0; scaler = 1; w = 0; mask = 0; in_word = 0; bits = 0; ones = 0; k_end = 0;
  }
  // more words were consumed than the block holds ("Mismatch between bit set and decoded values")
  __device__ __forceinline__ bool exhausted() const { return bs.k > k_end; }
  // Restart points (SkipEntry): the state after some number of next() calls, and a cursor re-entered there.
  __device__ __forceinline__ SkipEntry save(const PageView &pv) const {
    SkipEntry e;
    e.v = v;
    e.a = bs.k - bs.first_word_index(pv.data + 10);
    e.b = in_word;
    return e;
  }
  __device__ __forceinline__ void restore(const PageView &pv, uint32_t lane_ring, const SkipEntry &e) {
    const uint8_t *d = pv.data;
    scaler = ZZ ? 1 : pow10_u64(__ldg(d + 1) & 0xf);
    v = e.v;
    bs.init_at(d + 10, lane_ring, d + pv.data_len, e.a);
    k_end = bs.first_word_index(d + 10) + ((pv.data_len - 10) >> 3);
    w = 0; mask = 0; bits = 0; ones = 0;
    in_word = e.b;
    if (e.a) {  // inside packed word e.a - 1: re-read it and drop the values already consumed
      const uint64_t full = load_be64(d + 10 + (size_t)(e.a - 1) * 8);
      const uint32_t sel = (uint32_t)(full >> 60);
      uint32_t count;
      s8b_lut(sel, count, bits);
      ones = sel < 2 ? 1u : 0u;
      mask = bits ? (~0ull >> (64 - bits)) : 0ull;
      w = full >> (bits * (count - in_word));  // <= 60
    }
  }

  __device__ __forceinline__ void refill() {
    if (in_word == 0) {
      w = bs.next();
      const uint32_t sel = (uint32_t)(w >> 60);
      if (sel == 15) {  // 1 x 60 bits
        in_word = 1; bits = 60; ones = 0; mask = 0x0fffffffffffffffull;
      } else {
        s8b_lut(sel, in_word, bits);
        ones = sel < 2 ? 1u : 0u;
        mask = bits ? (~0ull >> (64 - bits)) : 0ull;
      }
    }
    in_word--;
  }
  __device__ __forceinline__ uint64_t next() {
    refill();
    const uint64_t u = (w & mask) | ones;
    w >>= bits;  // bits <= 60
    v += ZZ ? (uint64_t)zigzag_dec(u) : u * scaler;
    return v;
  }
  // next() in 32-bit arithmetic (ZZ only), for pages whose values all sign-extend from their low 32 bits: returns the
  // value's low word. The running value's low word is the sum of the deltas' low words mod 2^32, and the low word of
  // zigzag_dec(u) depends only on bits 0..32 of u (a 60-bit code included). The high word of `v` goes stale.
  __device__ __forceinline__ uint32_t next32() {
    static_assert(ZZ, "next32: zig-zag deltas only");
    refill();
    const uint32_t lo = ((uint32_t)w & (uint32_t)mask) | ones;
    const uint32_t b32 = (uint32_t)(w >> 32) & (uint32_t)(mask >> 32);  // bit 32 of the code
    w >>= bits;
    const uint32_t v32 = (uint32_t)v + (__funnelshift_r(lo, b32, 1) ^ (0u - (lo & 1u)));
    v = (v & 0xffffffff00000000ull) | v32;
    return v32;
  }
};

// ------------------------------------------------------------------------------------------------
// Gorilla cursor (float.rs:418-606): MSB-first bit stream after id | 0x10 | first(8).
// Terminates on the sentinel 0x7ff8_0000_0000_00ff (float.rs:16). Like DeltaCursor, the first next()
// needs no special case: a fake "repeat" control bit is queued in front of the stream.
// ------------------------------------------------------------------------------------------------
template <typename STREAM = BeStream>
struct GorillaCursor {
  STREAM bs;
  uint64_t val;
  uint64_t hi, lo;     // 128-bit window of the MSB-first bit stream; `pos` bits of hi are consumed
  uint32_t pos;        // 0..63
  uint32_t bits_used;  // bits consumed so far (incl. the fake one)
  uint32_t bits_total; // (data_len - 10) * 8 + 1
  uint32_t trailing, meaningful;
  bool done, err;      // done: sentinel reached or error; err: stream ended before the sentinel

  __device__ inline tskv_status open(const PageView &pv, uint32_t smem_slot = 0) {
    done = false;
    err = false;
    trailing = 0;
    meaningful = 64;
    const uint8_t *d = pv.data;
    bs.init(d + 2, smem_slot, d + pv.data_len);
    val = bs.next();
    hi = 0;  // its last bit is the fake control bit 0 = "repeat the previous value"
    lo = bs.next();
    pos = 63;
    bits_used = 0;
    bits_total = (pv.data_len - 10) * 8 + 1;
    return TSKV_OK;
  }
  __device__ __forceinline__ bool consumed_any() const { return bits_used != 0; }

  // Next 64 bits of the stream, MSB-aligned, without consuming them.
  __device__ __forceinline__ uint64_t peek() const { return (hi << pos) | ((lo >> 1) >> (63 - pos)); }
  // Consumes n in [1,64] bits.
  __device__ __forceinline__ void skip(uint32_t n) {
    pos += n;
    bits_used += n;
    if (pos >= 64) {
      pos -= 64;
      hi = lo;
      lo = bs.next();
    }
  }

  // Decodes the next stream element; returns false at the sentinel / on error
  // ("unexpected end of block": the stream ended before the sentinel).
  __device__ __forceinline__ bool advance() {
    const uint32_t x = (uint32_t)(peek() >> 51);  // 13 bits: c0 c1 lead[5] sig[6]
    if (!(x & 0x1000)) {
      skip(1);  // repeat previous value: pushed without a sentinel test (float.rs:493-497), like the first value
      if (bits_used > bits_total) {
        err = true;
        return false;
      }
      return true;
    } else {
      if (!(x & 0x0800)) {
        skip(2);  // reuse the previous (leading, trailing) window
      } else {
        skip(13);
        const uint32_t leading = (x >> 6) & 0x1f;
        meaningful = x & 0x3f;
        if (meaningful > 0) {
          trailing = (uint8_t)(64 - leading - meaningful);  // u8 arithmetic like the reference
        } else {
          trailing = 0;
          meaningful = 64;
        }
      }
      const uint64_t s = peek() >> (64 - meaningful);
      skip(meaningful);
      val ^= s << (trailing & 0x3f);
    }
    if (bits_used > bits_total) {
      err = true;
      return false;
    }
    return val != 0x7ff80000000000ffull;
  }

  // Value for the next VALID row; sets `done` when the stream ended before the bitset did.
  __device__ __forceinline__ uint64_t next() {
    if (done || !advance()) done = true;
    return val;
  }
  // The reference decodes to the sentinel (float.rs:480-591): a stream without one is an error even
  // when enough values were produced. Returns false on "unexpected end of block".
  __device__ __forceinline__ bool drain() {
    while (!done) {
      if (!advance()) done = true;
    }
    return !err;
  }
};

// ------------------------------------------------------------------------------------------------
// Gorilla cursor of the fused scan (float.rs:418-606), round 2: same results as GorillaCursor above, different
// mechanics. The bit stream is staged through a ChunkRing and addressed by absolute bit position: one element is
//   three 8-byte LDS (a 128-bit window at `pos`), a branch-free parse of the 13 control bits
//   (c0 c1 leading[5] meaningful[6]), two funnel shifts for the XOR payload, pos += len + sig
// with no per-lane branches: the 32 lanes of a warp decode 32 different pages and would diverge on every element.
// The cursor runs ONE ELEMENT AHEAD: next() returns the value decoded by the previous call and decodes the following
// element, so the first call needs no special case and the caller's arithmetic overlaps the next element's dependent
// chain. `cur_ok` says whether the value about to be returned is a real one (not the sentinel 0x7ff8_0000_0000_00ff,
// float.rs:16, and inside the block); asking for a value that is not sets the sticky `done` like the serial cursor.
// ------------------------------------------------------------------------------------------------
struct GorillaRing {
  ChunkRing ring;
  uint64_t val;         // value the next call returns
  uint32_t pos;         // bit position of the next element (ring coordinates)
  uint32_t end_pos;     // bit position of the end of the block
  uint32_t meaningful, trailing;
  bool cur_ok;          // `val` is a real value (not the terminating sentinel)
  bool done;            // a value was asked for after the sentinel
  bool any;

  __device__ __forceinline__ void open(const PageView &pv, uint32_t lane_slot) {
    const uint8_t *d = pv.data;  // id | 0x10 | first(8) | bit stream
    val = load_be64(d + 2);
    ring.init(d + 10, d + pv.data_len, lane_slot);
    pos = start_pos(d);
    end_pos = pos + (pv.data_len - 10) * 8;
    meaningful = 64;
    trailing = 0;
    cur_ok = true;  // the first value is pushed without a sentinel test (float.rs:445-460)
    done = any = false;
  }
  __device__ __forceinline__ void reset(uint32_t lane_slot) {
    ring.reset(lane_slot);
    val = 0; pos = 0; end_pos = 0; meaningful = 64; trailing = 0;
    cur_ok = false; done = any = false;
  }
  __device__ __forceinline__ bool consumed_any() const { return any; }
  // ring-coordinate bit position of the stream's first bit (data = id | 0x10 | first(8) | bit stream)
  static __device__ __forceinline__ uint32_t start_pos(const uint8_t *data) {
    return (uint32_t)(reinterpret_cast<uintptr_t>(data + 10) & 15) * 8 + ChunkRing::rot() * 128;
  }
  // Restart points (SkipEntry): the state before some next() call, and a cursor re-entered there.
  __device__ __forceinline__ SkipEntry save(const PageView &pv) const {
    SkipEntry e;
    e.v = val;
    e.a = pos - start_pos(pv.data);
    e.b = meaningful | (trailing << 8) | ((cur_ok ? 1u : 0u) << 16) | ((any ? 1u : 0u) << 17);
    return e;
  }
  __device__ __forceinline__ void restore(const PageView &pv, uint32_t lane_slot, const SkipEntry &e) {
    const uint8_t *d = pv.data;
    val = e.v;
    const uint32_t pos0 = start_pos(d);
    pos = pos0 + e.a;
    end_pos = pos0 + (pv.data_len - 10) * 8;
    ring.init_at(d + 10, d + pv.data_len, lane_slot, pos >> 7);
    meaningful = e.b & 0xff;
    trailing = (e.b >> 8) & 0xff;
    cur_ok = (e.b >> 16) & 1;
    any = (e.b >> 17) & 1;
    done = false;
  }
  // "unexpected end of block" (float.rs:462): an element ran past the block. `pos` only grows and stops growing at the
  // sentinel, so this one comparison, made when the caller checks, stands for the serial cursor's per-element test: an
  // overrun BEFORE the sentinel leaves pos > end_pos, a sentinel inside the block freezes pos <= end_pos.
  __device__ __forceinline__ bool overran() const { return pos > end_pos; }
  // Asked for more values than the stream holds, or the stream is truncated.
  __device__ __forceinline__ bool failed() const { return done || overran(); }

  // Decodes the element at `pos` into `val`.
  __device__ __forceinline__ void step() {
    ring.step(pos >> 7);
    const uint32_t k = pos >> 6;
    uint2 w0, w1, w2;
    ring.words3(k, w0, w1, w2);
    const bool up = pos & 32;  // the window starts in the upper half of w0
    const uint32_t a0 = __byte_perm(up ? w0.y : w0.x, 0, 0x0123), a1 = __byte_perm(up ? w1.x : w0.y, 0, 0x0123),
                   a2 = __byte_perm(up ? w1.y : w1.x, 0, 0x0123), a3 = __byte_perm(up ? w2.x : w1.y, 0, 0x0123);
    const uint32_t s = pos & 31;
    const uint32_t H = __funnelshift_l(a1, a0, s), M = __funnelshift_l(a2, a1, s), L = __funnelshift_l(a3, a2, s);
    const uint32_t x = H >> 19;  // 13 bits: c0 c1 leading[5] meaningful[6]
    const bool c0 = x & 0x1000, c1 = x & 0x0800;
    const uint32_t leading = (x >> 6) & 0x1f, m = x & 0x3f;
    const bool fresh = c0 && c1;
    meaningful = fresh ? (m ? m : 64u) : meaningful;
    trailing = fresh ? (m ? ((64u - leading - m) & 0xffu) : 0u) : trailing;  // u8 arithmetic like the reference
    const uint32_t len = c0 ? (c1 ? 13u : 2u) : 1u;
    const uint32_t sig = c0 ? meaningful : 0u;
    const uint64_t payload = ((uint64_t)__funnelshift_l(M, H, len) << 32) | __funnelshift_l(L, M, len);
    // shr.b64 / shl.b64 clamp the shift amount at 64: a repeat element (sig = 0) shifts everything out, delta = 0
    uint64_t delta;
    asm("{\n\t.reg .b64 t;\n\tshr.b64 t, %1, %2;\n\tshl.b64 %0, t, %3;\n\t}" : "=l"(delta) : "l"(payload), "r"(64u - sig), "r"(trailing & 63u));
    val ^= delta;
    pos += cur_ok ? len + sig : 0u;  // frozen once the sentinel has been seen (the lane keeps re-reading it, harmlessly)
    // the sentinel ends the stream (float.rs:585-589); repeats are pushed without the test (float.rs:493-497)
    cur_ok = cur_ok && !(c0 && val == 0x7ff80000000000ffull);
  }
  // Value for the next VALID row; sets `done` when the stream ended before the bitset did.
  __device__ __forceinline__ uint64_t next() {
    const uint64_t r = val;
    done = done || !cur_ok;
    any = true;
    step();
    return r;
  }
  // The reference decodes to the sentinel (float.rs:480-591): a stream without one is an error even when enough
  // values were produced. Returns false on "unexpected end of block".
  __device__ __forceinline__ bool drain() {
    while (!done && cur_ok && !overran()) step();
    return !overran();
  }
};

// Runtime-dispatched cursor over every supported kind (decode-only kernel).
template <typename STREAM = BeStream>
struct AnyCursor {
  DeltaCursor<-1, STREAM> d;
  GorillaCursor<STREAM> g;
  bool is_gorilla;
  __device__ inline tskv_status open(const PageView &pv, uint8_t kind, uint32_t smem_slot = 0) {
    is_gorilla = kind == DK_GORILLA;
    if (is_gorilla) return g.open(pv, smem_slot);
    return d.open(pv, kind, smem_slot);
  }
  __device__ __forceinline__ uint64_t next() { return is_gorilla ? g.next() : d.next(); }
  // more valid rows than encoded values (BITSET_MISMATCH) / truncated stream (SHORT_BLOCK)
  __device__ __forceinline__ bool failed() const { return is_gorilla ? g.done : d.exhausted; }
  __device__ __forceinline__ bool stream_error() const { return is_gorilla && g.err; }
};

// Error status a page kind maps to before any decoding (host classification).
__device__ __forceinline__ tskv_status kind_status(uint8_t kind) {
  switch (kind) {
    case DK_BAD_ENCODING: return TSKV_ERR_BAD_ENCODING;
    case DK_UNSUPPORTED: return TSKV_ERR_UNSUPPORTED;
    case DK_SHORT: return TSKV_ERR_SHORT_BLOCK;
    case DK_BAD_LENGTH: return TSKV_ERR_BAD_LENGTH;
    case DK_BAD_PAGE: return TSKV_ERR_PAGE_FORMAT;
    default: return TSKV_OK;
  }
}

}  // namespace tskv
