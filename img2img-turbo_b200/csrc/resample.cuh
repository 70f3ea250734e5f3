// LANCZOS resize of uint8 RGB images, bit-exact with PIL's Image.resize(size, Image.LANCZOS) (default box, no reducing_gap):
// what the reference CLIs run on the host before and after the forward (src/inference_unpaired.py:40-45,53;
// src/inference_paired.py:38-41).  PIL resizes in two separable passes, horizontal first, each rounding and clipping to
// uint8 on its own; a pass runs only when its dimension changes.
//
// The coefficient tables are computed on the HOST, in double, with the C library's sin (the function PIL calls), then
// uploaded once per plan: device sin differs in the last bits, and a last-bit difference can move a fixed-point rounding.
#pragma once
#include <cmath>
#include <map>
#include <memory>
#include <utility>
#include <vector>

#include "common.cuh"

namespace i2it {

constexpr int RS_PRECISION_BITS = 22;

struct ResampleTable {
  int ksize = 0;
  std::vector<int> bounds;   // [out][2]: first input index, number of taps
  std::vector<int> coeffs;   // [out][ksize]: 22-bit fixed-point weights, zero past the taps
};

inline double rs_sinc(double x) {
  if (x == 0.0) return 1.0;
  x = x * M_PI;
  return std::sin(x) / x;
}
inline double rs_lanczos(double x) { return (-3.0 <= x && x < 3.0) ? rs_sinc(x) * rs_sinc(x / 3) : 0.0; }

// One pass from `in` to `out` samples.  Each output index i has its own window of taps around (i + 0.5) * in / out, so a
// crop of the resized image is the same table restricted to the cropped indices.
inline ResampleTable lanczos_table(int in, int out) {
  I2IT_CHECK(in > 0 && out > 0, "resample: sizes must be positive");
  const double scale = static_cast<double>(in) / out;
  const double fs = scale < 1.0 ? 1.0 : scale;            // downscaling widens the filter by the scale
  const double support = 3.0 * fs, ss = 1.0 / fs;
  ResampleTable t;
  t.ksize = static_cast<int>(std::ceil(support)) * 2 + 1;
  t.bounds.resize(2 * static_cast<size_t>(out));
  t.coeffs.assign(static_cast<size_t>(out) * t.ksize, 0);
  std::vector<double> w(t.ksize);
  const double one = static_cast<double>(1 << RS_PRECISION_BITS);
  for (int i = 0; i < out; ++i) {
    const double center = (i + 0.5) * scale;
    int xmin = static_cast<int>(center - support + 0.5);
    if (xmin < 0) xmin = 0;
    int xmax = static_cast<int>(center + support + 0.5);
    if (xmax > in) xmax = in;
    const int n = xmax - xmin;
    double ww = 0.0;
    for (int x = 0; x < n; ++x) {
      w[x] = rs_lanczos((x + xmin - center + 0.5) * ss);
      ww += w[x];
    }
    int* k = t.coeffs.data() + static_cast<size_t>(i) * t.ksize;
    long long abs_sum = 0;
    for (int x = 0; x < n; ++x) {
      const double v = ww != 0.0 ? w[x] / ww : w[x];
      k[x] = v < 0 ? static_cast<int>(v * one - 0.5) : static_cast<int>(v * one + 0.5);
      abs_sum += k[x] < 0 ? -static_cast<long long>(k[x]) : k[x];
    }
    // The passes accumulate in int32 from 2^21, so every partial sum satisfies |acc| <= 2^21 + 255 * sum|k|.  The weights
    // of a row sum to 2^22 and the negative lobes are small: sum|k| < 1.6 * 2^22 for every size pair the tests sweep,
    // which bounds |acc| by 0.79 * 2^31.  A row that could overflow is refused here, before any launch.
    I2IT_CHECK((1ll << (RS_PRECISION_BITS - 1)) + 255 * abs_sum < (1ll << 31), "resample: int32 accumulator could overflow");
    t.bounds[2 * static_cast<size_t>(i)] = xmin;
    t.bounds[2 * static_cast<size_t>(i) + 1] = n;
  }
  return t;
}

__device__ __forceinline__ uint8_t rs_clip8(int acc) {
  const int v = acc >> RS_PRECISION_BITS;
  return static_cast<uint8_t>(v < 0 ? 0 : (v > 255 ? 255 : v));
}

// One output pixel of a pass: n taps k[0 .. n) over the RGB pixels s, s + step, s + 2 step, ... (step 3 along a row, the row
// pitch down a column), accumulated in int32 from 2^21, rounded and clipped to uint8.  Every pass, fixed or ragged, runs this.
__device__ __forceinline__ void rs_taps(const uint8_t* __restrict__ s, long long step, const int* __restrict__ k, int n,
                                        uint8_t* __restrict__ d) {
  int a0 = 1 << (RS_PRECISION_BITS - 1), a1 = a0, a2 = a0;
  for (int t = 0; t < n; ++t) {
    const int c = __ldg(k + t);
    const uint8_t* q = s + t * step;
    a0 += c * q[0];
    a1 += c * q[1];
    a2 += c * q[2];
  }
  d[0] = rs_clip8(a0); d[1] = rs_clip8(a1); d[2] = rs_clip8(a2);
}

// ------------------------------------------------------------------------------------------ the passes
// A launch runs one pass over a list of images, each with its own descriptor in device memory.  Its blocks stride over the
// launch's output rows (image by image: item0 counts the rows of the images before), so the grid need not depend on the
// images and a ragged plan's one captured graph serves any mix of sizes.
//
// One image of one pass: `rows` output rows of `cols` pixels.  Its table, at `tab` ints into the table area, holds the
// window's outputs only: bounds [outputs][2] (first source index, taps) then coefficients [outputs][ksize].
//   horizontal: output row r is source row row0 + r; output column j takes table row j
//   vertical:   output row r takes table row r and reads source rows from bounds[r].first - row0 (the horizontal pass made
//               only the rows from row0 on); output column j is source column j
// src and dst are relative to the launch's src_base / dst_base.  A ragged launch passes 0: its descriptors, uploaded with
// every call, hold the images' addresses.  A fixed plan passes the caller's pointer, read at launch: its descriptors,
// uploaded once, hold each image's offset from it.
struct RsPass {
  uintptr_t src, dst;
  long long src_pitch, dst_pitch;   // bytes per row
  long long tab;
  long long item0;
  int rows, cols, ksize, row0;
};

// the image whose rows hold work item `it`: the last one with item0 <= it (item0 ascends from 0)
__device__ __forceinline__ int rs_image_of(const RsPass* __restrict__ d, int n, long long it) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (d[mid].item0 <= it) lo = mid; else hi = mid - 1;
  }
  return lo;
}

static __global__ void resample_h_kernel(const RsPass* __restrict__ d, int n, const int* __restrict__ tab, uintptr_t src_base,
                                         uintptr_t dst_base) {
  pdl_sync();
  const long long total = d[n - 1].item0 + d[n - 1].rows;
  for (long long it = blockIdx.x; it < total; it += gridDim.x) {
    const RsPass p = d[rs_image_of(d, n, it)];
    const long long r = it - p.item0;
    const int* bounds = tab + p.tab;
    const int* coeffs = bounds + 2ll * p.cols;
    const uint8_t* s = reinterpret_cast<const uint8_t*>(src_base + p.src) + (p.row0 + r) * p.src_pitch;
    uint8_t* o = reinterpret_cast<uint8_t*>(dst_base + p.dst) + r * p.dst_pitch;
    for (int j = threadIdx.x; j < p.cols; j += blockDim.x)
      rs_taps(s + 3ll * bounds[2 * j], 3, coeffs + static_cast<long long>(j) * p.ksize, bounds[2 * j + 1], o + 3ll * j);
  }
}

static __global__ void resample_v_kernel(const RsPass* __restrict__ d, int n, const int* __restrict__ tab, uintptr_t src_base,
                                         uintptr_t dst_base) {
  pdl_sync();
  const long long total = d[n - 1].item0 + d[n - 1].rows;
  for (long long it = blockIdx.x; it < total; it += gridDim.x) {
    const RsPass p = d[rs_image_of(d, n, it)];
    const int r = static_cast<int>(it - p.item0);
    const int* bounds = tab + p.tab;
    const int* k = bounds + 2ll * p.rows + static_cast<long long>(r) * p.ksize;
    const int taps = bounds[2 * r + 1];
    const uint8_t* s = reinterpret_cast<const uint8_t*>(src_base + p.src) + static_cast<long long>(bounds[2 * r] - p.row0) * p.src_pitch;
    uint8_t* o = reinterpret_cast<uint8_t*>(dst_base + p.dst) + r * p.dst_pitch;
    for (int j = threadIdx.x; j < p.cols; j += blockDim.x) rs_taps(s + 3ll * j, p.src_pitch, k, taps, o + 3ll * j);
  }
}

// ---- host side ----
// lanczos_table per (in, out) pair, kept across calls: building one calls sin for every tap
class RsTableCache {
 public:
  std::shared_ptr<const ResampleTable> get(int in, int out) {
    auto it = m_.find({in, out});
    if (it != m_.end()) return it->second;
    if (m_.size() >= 512) m_.clear();
    auto t = std::make_shared<const ResampleTable>(lanczos_table(in, out));
    m_[{in, out}] = t;
    return t;
  }
 private:
  std::map<std::pair<int, int>, std::shared_ptr<const ResampleTable>> m_;
};

// Table ints of one ragged pass of `win` outputs from `in` samples: 2 bounds per output plus ksize coefficients, where
// ksize = 2 ceil(3 fs) + 1 with fs = max(in / out, 1) and out >= win the resized size.  Downscaling, ceil(3 fs) <= 3 fs + 1
// gives ksize <= 6 in / out + 3, so ksize win <= 6 in + 3 win; upscaling, ksize = 7; an identity pass has ksize 1.  Hence
// at most 2 win + max(6 in + 3 win, 7 win) <= 6 in + 9 win, monotone in both, so capacities bound every call.
inline long long rs_pass_bound(long long in, long long win) { return 6 * in + 9 * win; }

// table area of a ragged forward plan of B images on an H x W network with capacity max_side: per image, the input side's
// passes (from at most max_side to W columns and H rows) and the output side's (from W columns and H rows to at most max_side)
inline long long rs_forward_bound(long long B, long long H, long long W, long long max_side) {
  return B * (rs_pass_bound(max_side, W) + rs_pass_bound(max_side, H) + rs_pass_bound(W, max_side) + rs_pass_bound(H, max_side));
}

// One image of a resize: src [inH, inW, 3] resized to rsH x rsW, window (y0, x0, H, W) written densely to dst [H, W, 3];
// mid holds its horizontal pass's rows [rows, W, 3].  Addresses, or offsets from a launch's base (RsPass).
struct RsImage {
  uintptr_t src, dst, mid;
  int inH, inW, rsH, rsW, y0, x0, H, W;
};

// source rows [r0, r1) the vertical pass of `m` reads: what its horizontal pass makes
inline std::pair<int, int> rs_rows(const RsImage& m, RsTableCache& cache) {
  if (m.inH == m.rsH) return {m.y0, m.y0 + m.H};
  const auto t = cache.get(m.inH, m.rsH);
  const size_t last = 2 * static_cast<size_t>(m.y0 + m.H - 1);
  return {t->bounds[2 * static_cast<size_t>(m.y0)], t->bounds[last] + t->bounds[last + 1]};
}

// Appends the window [first, first + count) of the (in -> out) table to `tab`; returns its offset and sets ksize.  With
// in == out it is the identity: one tap of weight 1 << 22 per output, and (2^21 + v 2^22) >> 22 == v, the bytes PIL keeps
// when it skips the pass.
inline long long rs_put_table(std::vector<int>& tab, RsTableCache& cache, int in, int out, int first, int count, int* ksize) {
  const long long off = static_cast<long long>(tab.size());
  if (in == out) {
    *ksize = 1;
    for (int j = 0; j < count; ++j) { tab.push_back(first + j); tab.push_back(1); }
    tab.insert(tab.end(), count, 1 << RS_PRECISION_BITS);
    return off;
  }
  const auto t = cache.get(in, out);
  *ksize = t->ksize;
  tab.insert(tab.end(), t->bounds.begin() + 2 * static_cast<size_t>(first), t->bounds.begin() + 2 * static_cast<size_t>(first + count));
  tab.insert(tab.end(), t->coeffs.begin() + static_cast<size_t>(first) * t->ksize,
             t->coeffs.begin() + static_cast<size_t>(first + count) * t->ksize);
  return off;
}

// Appends the passes of n images of geometry m to h and v, and their tables, once, to tab.  Image b reads m.src + b src_img,
// writes m.dst + b dst_img and keeps its horizontal pass's rows at m.mid + b times their bytes.  bytes[0] / bytes[1] accumulate
// the passes' algorithmic bytes (pixels read and written, tables read once).  A ragged launch runs both passes for every
// image, an unchanged dimension as the identity.  With skip_identity a pass whose dimension does not change is left out, as
// PIL leaves it out: the other pass then reads the source (at column x0) or writes the destination itself.
inline void rs_add_images(const RsImage& m, int n, long long src_img, long long dst_img, bool skip_identity, RsTableCache& cache,
                          std::vector<RsPass>& h, std::vector<RsPass>& v, std::vector<int>& tab, double bytes[2]) {
  const std::pair<int, int> rr = rs_rows(m, cache);
  const bool need_h = !skip_identity || m.inW != m.rsW, need_v = !skip_identity || m.inH != m.rsH;
  const int rows = rr.second - rr.first;
  const long long mid_img = 3ll * rows * m.W;
  RsPass ph{}, pv{};
  if (need_v) pv.tab = rs_put_table(tab, cache, m.inH, m.rsH, m.y0, m.H, &pv.ksize);
  if (need_h) {
    ph.tab = rs_put_table(tab, cache, m.inW, m.rsW, m.x0, m.W, &ph.ksize);
    const int* hb = tab.data() + ph.tab;
    const long long span = hb[2 * (m.W - 1)] + hb[2 * (m.W - 1) + 1] - hb[0];
    ph.src = m.src; ph.src_pitch = 3ll * m.inW; ph.row0 = rr.first; ph.rows = rows; ph.cols = m.W;
    ph.dst = need_v ? m.mid : m.dst; ph.dst_pitch = 3ll * m.W;
    bytes[0] += 3.0 * n * rows * (span + m.W) + 4.0 * m.W * (2 + ph.ksize);
  }
  if (need_v) {
    pv.src = need_h ? m.mid : m.src + 3ll * m.x0; pv.src_pitch = need_h ? 3ll * m.W : 3ll * m.inW;
    pv.row0 = need_h ? rr.first : 0; pv.rows = m.H; pv.cols = m.W;
    pv.dst = m.dst; pv.dst_pitch = 3ll * m.W;
    bytes[1] += 3.0 * n * m.W * (rows + m.H) + 4.0 * m.H * (2 + pv.ksize);
  }
  for (long long b = 0; b < n; ++b) {
    if (need_h) {
      RsPass p = ph;
      p.src += b * src_img; p.dst += b * (need_v ? mid_img : dst_img);
      p.item0 = h.empty() ? 0 : h.back().item0 + h.back().rows;
      h.push_back(p);
    }
    if (need_v) {
      RsPass p = pv;
      p.src += b * (need_h ? mid_img : src_img); p.dst += b * dst_img;
      p.item0 = v.empty() ? 0 : v.back().item0 + v.back().rows;
      v.push_back(p);
    }
  }
}

}  // namespace i2it
