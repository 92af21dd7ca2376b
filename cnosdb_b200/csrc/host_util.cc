// host_util.cc — see host_util.h.
#include "host_util.h"

#include <algorithm>
#include <cmath>
#include <vector>
#include <mutex>

namespace tskv {

namespace {
uint32_t g_tab[8][256];
std::once_flag g_once;
void init_tables() {
  for (uint32_t i = 0; i < 256; i++) {
    uint32_t c = i;
    for (int k = 0; k < 8; k++) c = (c >> 1) ^ (0xEDB88320u & (0u - (c & 1)));
    g_tab[0][i] = c;
  }
  for (uint32_t i = 0; i < 256; i++)
    for (int t = 1; t < 8; t++) g_tab[t][i] = (g_tab[t - 1][i] >> 8) ^ g_tab[0][g_tab[t - 1][i] & 0xff];
}
inline uint32_t rd32be(const uint8_t *p) {
  return ((uint32_t)p[0] << 24) | ((uint32_t)p[1] << 16) | ((uint32_t)p[2] << 8) | p[3];
}
}  // namespace

const uint32_t *crc32_tables() {
  std::call_once(g_once, init_tables);
  return &g_tab[0][0];
}

uint32_t crc32_ieee(const uint8_t *p, size_t len) {
  std::call_once(g_once, init_tables);
  uint32_t crc = ~0u;
  while (len >= 8) {
    uint32_t lo = (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24);
    uint32_t hi = (uint32_t)p[4] | ((uint32_t)p[5] << 8) | ((uint32_t)p[6] << 16) | ((uint32_t)p[7] << 24);
    lo ^= crc;
    crc = g_tab[7][lo & 0xff] ^ g_tab[6][(lo >> 8) & 0xff] ^ g_tab[5][(lo >> 16) & 0xff] ^
          g_tab[4][lo >> 24] ^ g_tab[3][hi & 0xff] ^ g_tab[2][(hi >> 8) & 0xff] ^
          g_tab[1][(hi >> 16) & 0xff] ^ g_tab[0][hi >> 24];
    p += 8;
    len -= 8;
  }
  while (len--) crc = (crc >> 8) ^ g_tab[0][(crc ^ *p++) & 0xff];
  return ~crc;
}

double plan_selected_fraction(const uint32_t *arena_series, uint64_t n_arena, const uint32_t *sel, uint64_t n_sel) {
  if (!sel || n_arena == 0) return 1.0;
  const uint32_t *ie = sel + n_sel;
  const uint64_t in_range = (uint64_t)(std::upper_bound(sel, ie, arena_series[n_arena - 1]) - std::lower_bound(sel, ie, arena_series[0]));
  return std::min(1.0, (double)in_range / (double)n_arena);
}

void plan_serial_grids(int n_bins, const double *chunks, const double *t_chunk, const int *occ, int sm_count,
                       int warps_per_block, int *grid_out) {
  std::vector<double> cand;
  for (int b = 0; b < n_bins; b++) {
    grid_out[b] = 0;
    if (chunks[b] <= 0) continue;
    for (int k = 1; k <= 64; k++) cand.push_back(k * t_chunk[b]);
  }
  if (cand.empty()) return;
  std::sort(cand.begin(), cand.end());
  auto blocks_for = [&](int b, double T) -> double {
    const double rounds = std::floor(T / t_chunk[b] + 1e-9);
    if (rounds < 1) return -1;
    return std::ceil(chunks[b] / (rounds * warps_per_block));
  };
  double best = cand.back();
  for (double T : cand) {
    double sm_used = 0;
    bool ok = true;
    for (int b = 0; b < n_bins && ok; b++) {
      if (chunks[b] <= 0) continue;
      const double n = blocks_for(b, T);
      if (n < 0) ok = false;
      else sm_used += n / std::max(1, occ[b]);
    }
    if (ok && sm_used <= sm_count) { best = T; break; }
  }
  for (int b = 0; b < n_bins; b++)
    if (chunks[b] > 0) grid_out[b] = std::max(1, (int)std::max(1.0, blocks_for(b, best)));
}

uint32_t plan_parts_wanted(double est_chunks, double resident_warps, double target) {
  if (est_chunks <= 0) return 1;
  return (uint32_t)std::min(4096.0, std::max(1.0, std::ceil(target * resident_warps / est_chunks)));
}

uint32_t plan_bin_parts(uint32_t maxrows, uint32_t skip_rows, uint32_t want, uint32_t *part_rows) {
  *part_rows = 0;
  if (maxrows <= skip_rows || want <= 1) return 1;
  const uint32_t units = (maxrows + skip_rows - 1) / skip_rows;       // restart intervals of the longest page
  const uint32_t w = std::min(want, units);
  const uint32_t m = (units + w - 1) / w;                              // intervals per part
  *part_rows = m * skip_rows;
  return (units + m - 1) / m;
}

void plan_overlap_groups(uint64_t n_cg, const uint32_t *cg_series, const uint32_t *cg_rows, const tskv_time_range *cg_bounds,
                         const uint64_t *cg_file, OverlapPlan *out) {
  *out = OverlapPlan{};
  out->cg_merge.assign(n_cg, 0);
  out->mcg_row0.push_back(0);
  out->stream_first_mcg.push_back(0);
  out->group_first_stream.push_back(0);
  std::vector<uint32_t> order(n_cg);
  for (uint64_t i = 0; i < n_cg; i++) order[i] = (uint32_t)i;
  std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return cg_series[a] < cg_series[b]; });
  struct Chunk {
    uint64_t file;
    int64_t lo, hi;
    std::vector<uint32_t> cgs;
  };
  for (uint64_t i = 0; i < n_cg;) {
    uint64_t j = i;
    while (j < n_cg && cg_series[order[j]] == cg_series[order[i]]) j++;
    std::vector<Chunk> chunks;  // of this series
    for (uint64_t k = i; k < j; k++) {
      const uint32_t cg = order[k];
      Chunk *ch = nullptr;
      for (Chunk &c : chunks)
        if (c.file == cg_file[cg]) ch = &c;
      if (!ch) {
        chunks.push_back(Chunk{cg_file[cg], INT64_MAX, INT64_MIN, {}});
        ch = &chunks.back();
      }
      ch->lo = std::min(ch->lo, cg_bounds[cg].min_ts);
      ch->hi = std::max(ch->hi, cg_bounds[cg].max_ts);
      ch->cgs.push_back(cg);
    }
    i = j;
    if (chunks.size() == 1) {
      out->n_groups_total++;
      continue;
    }
    for (Chunk &c : chunks)  // a chunk's column groups in time order (tsm/chunk.rs:100-110 keeps them so)
      std::stable_sort(c.cgs.begin(), c.cgs.end(), [&](uint32_t a, uint32_t b) { return cg_bounds[a].min_ts < cg_bounds[b].min_ts; });
    std::sort(chunks.begin(), chunks.end(), [](const Chunk &a, const Chunk &b) {  // by time range, then file id
      if (a.lo != b.lo) return a.lo < b.lo;
      if (a.hi != b.hi) return a.hi < b.hi;
      return a.file < b.file;
    });
    size_t g0 = 0;
    int64_t run_max = INT64_MIN;
    auto close_group = [&](size_t a, size_t b) {  // chunks [a, b)
      out->n_groups_total++;
      if (b - a < 2) return;
      std::vector<const Chunk *> g;
      for (size_t k = a; k < b; k++) g.push_back(&chunks[k]);
      std::stable_sort(g.begin(), g.end(), [](const Chunk *x, const Chunk *y) { return x->file < y->file; });
      const uint32_t gi = (uint32_t)out->group_first_stream.size() - 1;
      for (const Chunk *c : g) {
        const uint32_t si = (uint32_t)out->stream_group.size();
        out->stream_group.push_back(gi);
        for (uint32_t cg : c->cgs) {
          out->cg_merge[cg] = 1;
          out->mcg_cg.push_back(cg);
          out->mcg_stream.push_back(si);
          out->mcg_row0.push_back(out->mcg_row0.back() + cg_rows[cg]);
        }
        out->stream_first_mcg.push_back((uint32_t)out->mcg_cg.size());
      }
      out->group_first_stream.push_back((uint32_t)out->stream_group.size());
    };
    for (size_t k = 0; k < chunks.size(); k++) {
      if (k > g0 && !(chunks[k].lo <= run_max)) {
        close_group(g0, k);
        g0 = k;
      }
      run_max = std::max(run_max, chunks[k].hi);
    }
    close_group(g0, chunks.size());
  }
}

bool parse_page(const uint8_t *page, uint64_t size, PageHeader *h) {
  if (size < 16) return false;
  h->bitset_len = rd32be(page);
  h->n_rows = ((uint64_t)rd32be(page + 4) << 32) | rd32be(page + 8);
  h->crc = rd32be(page + 12);
  if (16 + (uint64_t)h->bitset_len > size) return false;
  if ((uint64_t)h->bitset_len * 8 < h->n_rows) return false;
  h->bitset = page + 16;
  h->data = page + 16 + h->bitset_len;
  h->data_len = size - 16 - h->bitset_len;
  return true;
}

uint8_t classify_page(const PageHeader &h, uint8_t phys_type) {
  if (h.data_len == 0) return DK_ALLNULL;  // every codec: empty buffer => all-null array
  const uint8_t *d = h.data;
  unsigned enc = d[0];
  if (phys_type == TSKV_PT_BOOL) {  // get_bool_codec (instance.rs:415-421): Null => bytes, everything else => bit-pack
    if (enc == TSKV_ENC_NULL) return DK_BOOL_RAW;
    if (h.data_len < 3) return DK_SHORT;
    if (d[1] != 0x10) return DK_BAD_ENCODING;  // assert_eq!(src[0], BOOLEAN_COMPRESSED_BIT_PACKED << 4) (boolean.rs:84)
    uint64_t shift = 0;
    for (uint64_t i = 2; i < h.data_len; i++) {  // "boolean decoder: invalid count": the varint must end inside the block
      if ((d[i] & 0x80) == 0) return DK_BOOL_PACK;
      shift += 7;
      if (shift > 63) break;
    }
    return DK_SHORT;
  }
  if (enc == TSKV_ENC_QUANTILE) return DK_UNSUPPORTED;
  if (enc == TSKV_ENC_NULL) return ((h.data_len - 1) & 7) ? DK_BAD_LENGTH : DK_RAWBE;
  bool ts_family;
  switch (phys_type) {
    case TSKV_PT_TIME: ts_family = enc != TSKV_ENC_DELTA; break;      // get_ts_codec
    case TSKV_PT_I64: ts_family = enc == TSKV_ENC_DELTA_TS; break;    // get_i64_codec
    case TSKV_PT_U64: ts_family = false; break;                       // get_u64_codec
    case TSKV_PT_F64:                                                 // get_f64_codec => gorilla
      return h.data_len < 10 ? DK_SHORT : DK_GORILLA;
    default: return DK_UNSUPPORTED;
  }
  if (h.data_len < 2) return DK_SHORT;  // src[0] on an empty slice panics in the reference
  unsigned sub = d[1] >> 4;
  if (sub > 2) return DK_BAD_ENCODING;
  if (sub == 0) {
    uint64_t l = h.data_len - 2;
    if (l == 0 || (l & 7)) return DK_BAD_LENGTH;
    return ts_family ? DK_RAW_SC : DK_RAW_ZZ;
  }
  if (h.data_len < 10) return DK_SHORT;
  if (sub == 2) return ts_family ? DK_RLE_SC : DK_RLE_ZZ;
  if ((h.data_len - 10) & 7) return DK_SHORT;  // simple8b::decode would slice out of bounds
  return ts_family ? DK_S8B_SC : DK_S8B_ZZ;
}

}  // namespace tskv
