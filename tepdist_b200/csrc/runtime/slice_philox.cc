#include "runtime/slice_philox.h"

#include <cmath>
#include <functional>
#include <cstring>
#include <stdexcept>

namespace tepdist {

namespace {
struct Range { int64_t start, len; };  // along one dim: a union of strided pieces is expanded per period

// indices (as [start,len) pieces) of dim `d` kept after applying all levels that cut dim d
std::vector<Range> DimPieces(int64_t extent, const std::vector<DimStrategy>& levels, const std::vector<int>& ids, int d) {
  std::vector<Range> pieces = {{0, extent}};
  for (size_t l = 0; l < levels.size(); ++l) {
    const DimStrategy& s = levels[l];
    if (!s.is_split() || s.dim != d) continue;
    const int k = l < ids.size() ? ids[l] : 0;
    std::vector<Range> next;
    // current logical extent = sum of piece lengths; the split acts on that logical index space
    int64_t logical = 0;
    for (auto& p : pieces) logical += p.len;
    const int64_t stride = s.stride > 0 ? s.stride : logical;
    const int64_t chunk = stride / s.num;
    // walk logical positions period by period, map back to physical pieces
    auto emit = [&](int64_t lo, int64_t len) {  // logical [lo, lo+len)
      int64_t pos = 0;
      for (auto& p : pieces) {
        const int64_t a = std::max(lo, pos), b = std::min(lo + len, pos + p.len);
        if (a < b) next.push_back({p.start + (a - pos), b - a});
        pos += p.len;
      }
    };
    for (int64_t base = 0; base < logical; base += stride) emit(base + k * chunk, chunk);
    pieces = next;
  }
  return pieces;
}
}  // namespace

std::vector<int64_t> ShardShape(const std::vector<int64_t>& shape, const std::vector<DimStrategy>& levels) {
  std::vector<int64_t> s = shape;
  for (auto& l : levels)
    if (l.is_split()) s[l.dim] /= l.num;
  return s;
}

std::vector<std::pair<int64_t, int64_t>> SliceRuns(const std::vector<int64_t>& shape, const std::vector<DimStrategy>& levels,
                                                   const std::vector<int>& ids) {
  const int r = (int)shape.size();
  std::vector<std::vector<Range>> pieces(r);
  for (int d = 0; d < r; ++d) pieces[d] = DimPieces(shape[d], levels, ids, d);
  std::vector<int64_t> strides(r, 1);
  for (int d = r - 2; d >= 0; --d) strides[d] = strides[d + 1] * shape[d + 1];
  // innermost dims that are kept whole merge into longer runs
  int inner = r;  // first dim (from the right) that is cut
  int64_t inner_len = 1;
  while (inner > 0 && pieces[inner - 1].size() == 1 && pieces[inner - 1][0].len == shape[inner - 1]) {
    --inner;
    inner_len *= shape[inner];
  }
  std::vector<std::pair<int64_t, int64_t>> runs;
  if (r == 0) { runs.push_back({0, 1}); return runs; }
  // enumerate index pieces of dims [0, inner) ; the last cut dim contributes (start,len) pieces directly
  std::vector<int64_t> idx_off;  // offsets for the outer dims, expanded element-wise
  std::function<void(int, int64_t)> rec = [&](int d, int64_t off) {
    if (d == inner) { runs.push_back({off, inner_len}); return; }
    const bool last_cut = (d == inner - 1);
    for (auto& p : pieces[d]) {
      if (last_cut) {
        runs.push_back({off + p.start * strides[d], p.len * inner_len});
      } else {
        for (int64_t i = 0; i < p.len; ++i) rec(d + 1, off + (p.start + i) * strides[d]);
      }
    }
  };
  if (inner == 0) runs.push_back({0, inner_len});
  else rec(0, 0);
  return runs;
}

void SliceCopy(const uint8_t* src, uint8_t* dst, int64_t es, const std::vector<int64_t>& shape,
               const std::vector<DimStrategy>& levels, const std::vector<int>& ids) {
  int64_t o = 0;
  for (auto& run : SliceRuns(shape, levels, ids)) {
    std::memcpy(dst + o * es, src + run.first * es, (size_t)(run.second * es));
    o += run.second;
  }
}

// ---------------------------------------------------------------------------------------------- Philox4x32-10
namespace {
inline void PhiloxRound(uint32_t (&c)[4], uint32_t (&k)[2]) {
  const uint64_t p0 = (uint64_t)0xD2511F53u * c[0], p1 = (uint64_t)0xCD9E8D57u * c[2];
  const uint32_t n0 = (uint32_t)(p1 >> 32) ^ c[1] ^ k[0], n1 = (uint32_t)p1;
  const uint32_t n2 = (uint32_t)(p0 >> 32) ^ c[3] ^ k[1], n3 = (uint32_t)p0;
  c[0] = n0; c[1] = n1; c[2] = n2; c[3] = n3;
  k[0] += 0x9E3779B9u;
  k[1] += 0xBB67AE85u;
}
inline void Philox10(uint64_t seed, uint32_t (&c)[4]) {
  uint32_t k[2] = {(uint32_t)seed, (uint32_t)(seed >> 32)};
  for (int i = 0; i < 10; ++i) PhiloxRound(c, k);
}
inline void PhiloxBlock(uint64_t seed, uint64_t block, uint32_t attempt, uint32_t (&out)[4]) {
  uint32_t c[4] = {(uint32_t)block, (uint32_t)(block >> 32), attempt, 0u};
  Philox10(seed, c);
  for (int i = 0; i < 4; ++i) out[i] = c[i];
}
inline float U01(uint32_t x) { return (float)((x >> 8) + 0.5f) * (1.0f / 16777216.0f); }  // (0,1)
inline void BoxMuller(uint32_t a, uint32_t b, float* z0, float* z1) {
  const float u1 = U01(a), u2 = U01(b);
  const float r = std::sqrt(-2.0f * std::log(u1));
  const float t = 6.28318530717958647692f * u2;
  *z0 = r * std::cos(t);
  *z1 = r * std::sin(t);
}
inline float ElementValue(int kind, uint64_t seed, int64_t i, float mean, float stddev, float lo, float hi) {
  const uint64_t block = (uint64_t)i >> 2;
  const int lane = (int)(i & 3);
  for (uint32_t attempt = 0;; ++attempt) {
    uint32_t r[4];
    PhiloxBlock(seed, block, attempt, r);
    if (kind == 0) return lo + (hi - lo) * U01(r[lane]);
    float z[4];
    BoxMuller(r[0], r[1], &z[0], &z[1]);
    BoxMuller(r[2], r[3], &z[2], &z[3]);
    if (kind == 1) return mean + stddev * z[lane];
    if (std::fabs(z[lane]) <= 2.0f || attempt > 64) return mean + stddev * z[lane];  // truncated normal
  }
}
int KindOf(const std::string& k) { return k == "uniform" ? 0 : (k == "normal" ? 1 : 2); }
}  // namespace

void PhiloxFill(const std::string& kind, uint64_t seed, int64_t offset, int64_t n, float mean, float stddev, float lo, float hi,
                float* out) {
  const int k = KindOf(kind);
  for (int64_t i = 0; i < n; ++i) out[i] = ElementValue(k, seed, offset + i, mean, stddev, lo, hi);
}

std::vector<float> PhiloxFillShard(const std::string& kind, uint64_t seed, const std::vector<int64_t>& shape,
                                   const std::vector<DimStrategy>& levels, const std::vector<int>& ids, float mean, float stddev,
                                   float lo, float hi) {
  std::vector<float> out;
  for (auto& run : SliceRuns(shape, levels, ids)) {
    const size_t o = out.size();
    out.resize(o + (size_t)run.second);
    PhiloxFill(kind, seed, run.first, run.second, mean, stddev, lo, hi, out.data() + o);
  }
  return out;
}

void DropoutKeep(uint64_t seed, uint32_t step, uint32_t site, int thr, bool attention, const std::vector<int64_t>& shape,
                 const std::vector<int64_t>& start, const std::vector<int64_t>& len, uint8_t* out) {
  const int r = (int)shape.size();
  if (r == 0 || (int)start.size() != r || (int)len.size() != r || (attention && (r != 4 || shape[2] != shape[3])))
    throw std::invalid_argument("DropoutKeep: the box must have the global shape's rank ([B, H, S, S] for attention)");
  int64_t n = 1;
  for (int d = 0; d < r; ++d) {
    if (start[d] < 0 || len[d] < 0 || start[d] + len[d] > shape[d]) throw std::invalid_argument("DropoutKeep: box outside the shape");
    n *= len[d];
  }
  std::vector<int64_t> idx(start);   // global coordinates of the current element (row-major walk over the box)
  uint32_t c[4], last0 = 0, last1 = 0;
  bool have = false;
  for (int64_t e = 0; e < n; ++e) {
    uint32_t c0, c1, byte;
    if (attention) {
      const int64_t S = shape[2], q = idx[2], k = idx[3];
      c0 = (uint32_t)(((k >> 5) << 2) | ((k >> 1) & 3));
      c1 = (uint32_t)((idx[0] * shape[1] + idx[1]) * S + (q & ~int64_t(8)));
      byte = (uint32_t)(8 * ((q >> 3) & 1) + 2 * ((k >> 3) & 3) + (k & 1));
    } else {
      int64_t row = 0;
      for (int d = 0; d < r - 1; ++d) row = row * shape[d] + idx[d];
      const int64_t col = idx[r - 1];
      c0 = (uint32_t)(col >> 4);
      c1 = (uint32_t)row;
      byte = (uint32_t)(col & 15);
    }
    if (!have || c0 != last0 || c1 != last1) {
      c[0] = c0; c[1] = c1; c[2] = step; c[3] = site;
      Philox10(seed, c);
      last0 = c0; last1 = c1; have = true;
    }
    out[e] = ((c[byte >> 2] >> (8 * (byte & 3))) & 0xffu) >= (uint32_t)thr;
    for (int d = r - 1; d >= 0; --d) {
      if (++idx[d] < start[d] + len[d]) break;
      idx[d] = start[d];
    }
  }
}

}  // namespace tepdist
