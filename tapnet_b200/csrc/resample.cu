// Lanczos resize of uint8 RGB clips, bit for bit as PIL's 8-bit resampler
// (Image.resize(..., LANCZOS), what mediapy.resize_video does to uint8 frames and what
// tapvid/evaluation_datasets.py:41-45 resize_video calls).  DESIGN section 10, row f6.
//
// Per axis (in -> out): scale = in / out, fs = max(scale, 1), support = 3 fs,
// ksize = 2 ceil(support) + 1.  Output o reads inputs xmin .. xmin + n - 1 around
// centre (o + 0.5) scale with weights lanczos((i + xmin - centre + 0.5) * (1 / fs)), normalised by their
// sum in double, then rounded half away from zero to 22 fraction bits.  A pass is
// clamp((2^21 + sum src * k) >> 22, 0, 255) in int32.  The weights need sin(), so the host computes
// them in double with libm (tapir_lanczos_weights) and the kernels are integer only.
//
// Two launches: a horizontal pass (only if W != w) into a uint8 intermediate holding just the
// rows the vertical pass reads, then a vertical pass (only if H != h); a clip of the same size is
// copied.  One thread per output byte: the horizontal pass reads its taps 3 bytes apart within
// the row (the warp's windows overlap in L1), the vertical pass reads whole rows, coalesced.
#include <algorithm>
#include <cmath>
#include <vector>

#include "kernels.cuh"

namespace tapir {
namespace {

constexpr int kPrecisionBits = 22;
constexpr int kResizeThreads = 256;
constexpr int kMaxGridRows = 65535;

double sinc(double x) {
  if (x == 0.0) return 1.0;
  x = x * M_PI;
  return sin(x) / x;
}

double lanczos(double x) {
  if (-3.0 <= x && x < 3.0) return sinc(x) * sinc(x / 3);
  return 0.0;
}

struct Axis {
  double scale, ss, support;
  int ksize;
  Axis(int in, int out) {
    scale = (double)in / out;
    const double fs = scale < 1.0 ? 1.0 : scale;
    ss = 1.0 / fs;
    support = 3.0 * fs;
    ksize = (int)ceil(support) * 2 + 1;
  }
  // inputs xmin .. xmin + n - 1 of output o (and its centre)
  void bounds(int in, int o, int* xmin, int* n, double* center) const {
    *center = (o + 0.5) * scale;
    int lo = (int)(*center - support + 0.5);
    if (lo < 0) lo = 0;
    int hi = (int)(*center + support + 0.5);
    if (hi > in) hi = in;
    *xmin = lo;
    *n = hi - lo;
  }
};

__device__ __forceinline__ uint8_t clip8(int acc) {
  const int v = acc >> kPrecisionBits;
  return (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v));
}

// Horizontal pass: dst row r (of `rows` per frame) = source row row0 + r % rows of frame r / rows.
// A thread owns one byte e = 3 ox + c of the output row; its window is clamped to the source row.
__global__ void __launch_bounds__(kResizeThreads) lanczos_rows_kernel(
    const uint8_t* __restrict__ src, int W, long long src_frame_bytes, int row0, int rows,
    long long total_rows, const int* __restrict__ bounds, const int* __restrict__ taps, int ksize,
    uint8_t* __restrict__ dst, int w) {
  const int e = blockIdx.x * kResizeThreads + threadIdx.x;
  if (e >= w * 3) return;
  const int ox = e / 3, c = e - ox * 3;
  const int x0 = min(max(bounds[2 * ox], 0), W);
  const int n = min(min(max(bounds[2 * ox + 1], 0), W - x0), ksize);
  const int* k = taps + (long long)ox * ksize;
  for (long long r = blockIdx.y; r < total_rows; r += gridDim.y) {
    const long long f = r / rows;
    const uint8_t* p = src + f * src_frame_bytes + ((long long)(row0 + (r - f * rows)) * W + x0) * 3 + c;
    int acc = 1 << (kPrecisionBits - 1);
    for (int i = 0; i < n; ++i) acc += (int)p[3 * i] * __ldg(k + i);
    dst[r * w * 3 + e] = clip8(acc);
  }
}

// Vertical pass: output row oy of frame f from rows bounds[oy] - row0 ... of the frame's `rows`
// source rows (the intermediate, or the source itself when W == w).  row_bytes = 3 w.
__global__ void __launch_bounds__(kResizeThreads) lanczos_cols_kernel(
    const uint8_t* __restrict__ src, int row0, int rows, int row_bytes, int h, long long total_rows,
    const int* __restrict__ bounds, const int* __restrict__ taps, int ksize,
    uint8_t* __restrict__ dst) {
  const int e = blockIdx.x * kResizeThreads + threadIdx.x;
  if (e >= row_bytes) return;
  for (long long r = blockIdx.y; r < total_rows; r += gridDim.y) {
    const long long f = r / h;
    const int oy = (int)(r - f * h);
    const int y0 = min(max(bounds[2 * oy] - row0, 0), rows);
    const int n = min(min(max(bounds[2 * oy + 1], 0), rows - y0), ksize);
    const int* k = taps + (long long)oy * ksize;
    const uint8_t* p = src + (f * rows + y0) * row_bytes + e;
    int acc = 1 << (kPrecisionBits - 1);
    for (int i = 0; i < n; ++i) acc += (int)p[(long long)i * row_bytes] * __ldg(k + i);
    dst[r * row_bytes + e] = clip8(acc);
  }
}

dim3 row_grid(int row_bytes, long long total_rows) {
  return dim3((unsigned)ceil_div_ll(row_bytes, kResizeThreads),
              (unsigned)std::min<long long>(total_rows, kMaxGridRows));
}

}  // namespace

int lanczos_ksize(int in_size, int out_size) { return Axis(in_size, out_size).ksize; }

void lanczos_weights(int in_size, int out_size, int* bounds, int* taps) {
  const Axis ax(in_size, out_size);
  std::vector<double> k(ax.ksize);
  for (int o = 0; o < out_size; ++o) {
    int xmin, n;
    double center;
    ax.bounds(in_size, o, &xmin, &n, &center);
    double ww = 0.0;
    for (int i = 0; i < n; ++i) {
      k[i] = lanczos((i + xmin - center + 0.5) * ax.ss);
      ww += k[i];
    }
    int* kk = taps + (long long)o * ax.ksize;
    for (int i = 0; i < ax.ksize; ++i) {
      double v = i < n ? k[i] : 0.0;
      if (i < n && ww != 0.0) v /= ww;
      kk[i] = v < 0 ? (int)(-0.5 + v * (1 << kPrecisionBits)) : (int)(0.5 + v * (1 << kPrecisionBits));
    }
    bounds[2 * o] = xmin;
    bounds[2 * o + 1] = n;
  }
}

void lanczos_row_span(int H, int h, int* row0, int* rows) {
  const Axis ax(H, h);
  int x0, n0, x1, n1;
  double c;
  ax.bounds(H, 0, &x0, &n0, &c);
  ax.bounds(H, h - 1, &x1, &n1, &c);
  *row0 = x0;
  *rows = x1 + n1 - x0;
}

size_t resize_lanczos_u8_workspace_bytes(int frames, int H, int W, int h, int w) {
  if (H == h || W == w) return 0;
  int row0, rows;
  lanczos_row_span(H, h, &row0, &rows);
  return (size_t)frames * rows * w * 3;
}

int resize_lanczos_u8(const uint8_t* src, uint8_t* dst, int frames, int H, int W, int h, int w,
                      const int* x_bounds, const int* x_taps, int x_ksize, const int* y_bounds,
                      const int* y_taps, int y_ksize, uint8_t* ws, cudaStream_t s) {
  const long long out_bytes = (long long)frames * h * w * 3;
  ProfileScope ps("resize_lanczos_u8", s, 0.0, (double)frames * H * W * 3 + (double)out_bytes);
  if (H == h && W == w) {
    TAPIR_CUDA(cudaMemcpyAsync(dst, src, (size_t)out_bytes, cudaMemcpyDeviceToDevice, s));
    return kOk;
  }
  int row0 = 0, rows = H;  // the source rows the vertical pass reads: all, or those of the intermediate
  if (W != w && H != h) lanczos_row_span(H, h, &row0, &rows);
  const uint8_t* mid = src;
  if (W != w) {
    uint8_t* out = (H == h) ? dst : ws;
    const long long total = (long long)frames * rows;
    lanczos_rows_kernel<<<row_grid(w * 3, total), kResizeThreads, 0, s>>>(
        src, W, (long long)H * W * 3, row0, rows, total, x_bounds, x_taps, x_ksize, out, w);
    count_launch();
    TAPIR_LAUNCH_CHECK("lanczos_rows_kernel");
    mid = out;
  }
  if (H != h) {
    const long long total = (long long)frames * h;
    lanczos_cols_kernel<<<row_grid(w * 3, total), kResizeThreads, 0, s>>>(
        mid, row0, rows, w * 3, h, total, y_bounds, y_taps, y_ksize, dst);
    count_launch();
    TAPIR_LAUNCH_CHECK("lanczos_cols_kernel");
  }
  return kOk;
}

}  // namespace tapir
