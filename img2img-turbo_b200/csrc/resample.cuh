// LANCZOS resize of uint8 RGB images, bit-exact with PIL's Image.resize(size, Image.LANCZOS) (default box, no reducing_gap):
// what the reference CLIs run on the host before and after the forward (src/inference_unpaired.py:40-45,53;
// src/inference_paired.py:38-41).  PIL resizes in two separable passes, horizontal first, each rounding and clipping to
// uint8 on its own; a pass runs only when its dimension changes.
//
// The coefficient tables are computed on the HOST, in double, with the C library's sin (the function PIL calls), then
// uploaded once per plan: device sin differs in the last bits, and a last-bit difference can move a fixed-point rounding.
#pragma once
#include <cmath>
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

// Horizontal pass: dst [B, rows, Wo, 3] = src rows row0 .. row0+rows-1 resampled along x, output columns x0 .. x0+Wo-1 of
// the table (a crop window).  src: [B][img / (src_w*3)][src_w][3], img bytes per image.  One thread per output pixel.
static __global__ void resample_h_u8_kernel(const uint8_t* __restrict__ src, long long src_img, int src_w, int row0,
                                            uint8_t* __restrict__ dst, int rows, int Wo, int x0, const int* __restrict__ bounds,
                                            const int* __restrict__ coeffs, int ksize, long long total) {
  pdl_sync();
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;   // over B*rows*Wo
  if (i >= total) return;
  const int j = static_cast<int>(i % Wo);
  const long long br = i / Wo;
  const int r = static_cast<int>(br % rows);
  const long long b = br / rows;
  const int xo = x0 + j, xmin = bounds[2 * xo], n = bounds[2 * xo + 1];
  const int* k = coeffs + static_cast<long long>(xo) * ksize;
  const uint8_t* s = src + b * src_img + (static_cast<long long>(row0 + r) * src_w + xmin) * 3;
  int a0 = 1 << (RS_PRECISION_BITS - 1), a1 = a0, a2 = a0;
  for (int t = 0; t < n; ++t) {
    const int c = __ldg(k + t);
    a0 += c * s[3 * t];
    a1 += c * s[3 * t + 1];
    a2 += c * s[3 * t + 2];
  }
  uint8_t* d = dst + i * 3;
  d[0] = rs_clip8(a0); d[1] = rs_clip8(a1); d[2] = rs_clip8(a2);
}

// Vertical pass: dst [B, Ho, Wo, 3] = output rows y0 .. y0+Ho-1 of the table, read from src columns col0 .. col0+Wo-1;
// src row index = table row index - row_shift (the horizontal pass computed only the rows from row_shift on).
static __global__ void resample_v_u8_kernel(const uint8_t* __restrict__ src, long long src_img, int src_w, int col0,
                                            int row_shift, uint8_t* __restrict__ dst, int Ho, int Wo, int y0,
                                            const int* __restrict__ bounds, const int* __restrict__ coeffs, int ksize,
                                            long long total) {
  pdl_sync();
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;   // over B*Ho*Wo
  if (i >= total) return;
  const int j = static_cast<int>(i % Wo);
  const long long bh = i / Wo;
  const int h = static_cast<int>(bh % Ho);
  const long long b = bh / Ho;
  const int yo = y0 + h, ymin = bounds[2 * yo] - row_shift, n = bounds[2 * yo + 1];
  const int* k = coeffs + static_cast<long long>(yo) * ksize;
  const long long pitch = static_cast<long long>(src_w) * 3;
  const uint8_t* s = src + b * src_img + static_cast<long long>(ymin) * pitch + static_cast<long long>(col0 + j) * 3;
  int a0 = 1 << (RS_PRECISION_BITS - 1), a1 = a0, a2 = a0;
  for (int t = 0; t < n; ++t) {
    const int c = __ldg(k + t);
    const uint8_t* q = s + t * pitch;
    a0 += c * q[0];
    a1 += c * q[1];
    a2 += c * q[2];
  }
  uint8_t* d = dst + i * 3;
  d[0] = rs_clip8(a0); d[1] = rs_clip8(a1); d[2] = rs_clip8(a2);
}

}  // namespace i2it
