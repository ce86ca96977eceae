// Painting point tracks onto uint8 RGB frames, bit for bit as the reference's paint_point_track
// (tapnet/utils/viz_utils.py:47-124), the step after the path (DESIGN section 10, row f5).
//
// The reference pastes, for every visible point in index order, a (2r+2)^2 patch of a bilinearly
// shifted round icon into the frame: v = uint8(trunc((1 - p) v + p c)) in float64, truncated after
// every point.  Two launches:
//   * footprint: one thread per (point, frame) turns the strided tracks [N][T][2] (fp32 or fp64)
//     and visibles [N][T] into frame-major records [T][N]: the integer corner (x1, y1) of the
//     patch (kHidden for a point that does not paint) and the clamped centre in float64;
//   * tiles: one CTA per (frame, 32 x 32 output tile) scans the frame's records in index order,
//     compacts the points whose patch touches the tile into a shared list (ballot + a prefix over
//     the warps keeps index order) and folds every pixel over that list in registers.  Each pixel
//     is read once and written once; no atomics, so the output is deterministic.
#include <algorithm>
#include <climits>
#include <cmath>

#include "kernels.cuh"

namespace tapir {
namespace {

constexpr int kTile = 32;                          // output tile edge in pixels
constexpr int kPaintThreads = 256;                 // a thread owns one column, kRowsPerThread rows
constexpr int kWarps = kPaintThreads / 32;
constexpr int kRowsPerThread = kTile / kWarps;     // rows warp, warp + 8, warp + 16, warp + 24
constexpr int kListCap = 2 * kPaintThreads;        // hit-list entries per round
constexpr int kHidden = INT_MIN;                   // x1 of a point that does not paint

// A point of the hit list: the bilinear weights of its patch, the patch's top-left pixel and
// its colour.
struct PaintEntry {
  double wx1, wx2, wy1, wy2;  // x - x1, x1 + 1 - x, y - y1, y1 + 1 - y
  int x0, y0;                 // x1 - r - 1, y1 - r - 1
  uint32_t rgb;
  int pad;
};

__device__ __forceinline__ float add_half(float v) { return __fadd_rn(v, 0.5f); }
__device__ __forceinline__ double add_half(double v) { return __dadd_rn(v, 0.5); }

// The centre is track + 0.5 in the tracks' own dtype, then min(max(v, 0.0), size) as Python
// evaluates it (a NaN passes through both comparisons and is skipped: the reference leaves it
// undefined).
template <typename F>
__global__ void __launch_bounds__(256) paint_footprint_kernel(
    const F* __restrict__ tracks, const uint8_t* __restrict__ visibles, int T, int N, int H, int W,
    int2* __restrict__ box, double2* __restrict__ centre) {
  const long long total = (long long)T * N;
  for (long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x; k < total;
       k += (long long)gridDim.x * blockDim.x) {
    const long long i = k / T, t = k - i * T;  // k = i * T + t: coalesced reads of the tracks
    double x = (double)add_half(tracks[k * 2 + 0]);
    double y = (double)add_half(tracks[k * 2 + 1]);
    x = (0.0 > x) ? 0.0 : x;
    x = ((double)W < x) ? (double)W : x;
    y = (0.0 > y) ? 0.0 : y;
    y = ((double)H < y) ? (double)H : y;
    int2 b = make_int2(kHidden, kHidden);
    if (visibles[k] != 0 && !isnan(x) && !isnan(y)) b = make_int2((int)floor(x), (int)floor(y));
    box[t * N + i] = b;
    centre[t * N + i] = make_double2(x, y);
  }
}

// The reference's icon at integer offset (dy, dx) from its (off-by-one) centre:
//   1 - clip((dy^2 + dx^2 - r^2 / 2.0) / (2r * 0.15), 0, 1).
// Only a ring about 0.2 px wide takes the division; inside it the value is exactly 1, outside 0.
__device__ __forceinline__ double icon_value(double q, double half_r2, double scale) {
  const double d = __dsub_rn(q, half_r2);
  if (d <= 0.0) return 1.0;
  if (d >= scale) return 0.0;  // d / scale >= 1 (also r = 0: scale 0, the reference's x / 0 = inf)
  return __dsub_rn(1.0, __ddiv_rn(d, scale));
}

__device__ __forceinline__ double sq(int v) { return __dmul_rn((double)v, (double)v); }

__global__ void __launch_bounds__(kPaintThreads, 2) paint_tiles_kernel(
    const uint8_t* __restrict__ frames, uint8_t* __restrict__ out, int H, int W, int N, int r,
    int tiles_x, int tiles_per_frame, const int2* __restrict__ box,
    const double2* __restrict__ centre, const uint8_t* __restrict__ colors) {
  __shared__ PaintEntry list[kListCap];
  __shared__ int warp_hits[2][kWarps];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int t = blockIdx.x / tiles_per_frame, tile = blockIdx.x - t * tiles_per_frame;
  const int tx0 = (tile % tiles_x) * kTile, ty0 = (tile / tiles_x) * kTile;
  const size_t frame_off = (size_t)t * H * W * 3;

  // Pixels outside the frame get a coordinate no patch reaches (every patch row / column index is
  // taken as unsigned (p - p0) <= 2r + 1).
  const int px = (tx0 + lane < W) ? tx0 + lane : INT_MIN / 2;
  int py[kRowsPerThread];
  double v[kRowsPerThread][3];
#pragma unroll
  for (int k = 0; k < kRowsPerThread; ++k) {
    const int y = ty0 + warp + kWarps * k;
    py[k] = (y < H && px >= 0) ? y : INT_MIN / 2;
    if (py[k] >= 0) {
      const uint8_t* p = frames + frame_off + ((size_t)y * W + px) * 3;
      v[k][0] = p[0];
      v[k][1] = p[1];
      v[k][2] = p[2];
    } else {
      v[k][0] = v[k][1] = v[k][2] = 0.0;
    }
  }

  if (N > 0) {
    const int2* fbox = box + (size_t)t * N;
    const double2* fcentre = centre + (size_t)t * N;
    // A patch covers columns x1 - r - 1 .. x1 + r: it touches the tile iff x1 in [lo_x, hi_x].
    const int last_x = min(tx0 + kTile, W) - 1, last_y = min(ty0 + kTile, H) - 1;
    const int lo_x = tx0 - r, lo_y = ty0 - r;  // > kHidden: a hidden point never hits
    const int hi_x = (int)min((long long)last_x + r + 1, (long long)INT_MAX);
    const int hi_y = (int)min((long long)last_y + r + 1, (long long)INT_MAX);
    const unsigned last = 2u * r + 1u;  // patch rows / columns 0 .. 2r + 1
    const double half_r2 = __dmul_rn((double)r, (double)r) / 2.0;
    const double scale = __dmul_rn((double)(2 * r), 0.15);

    int count = 0, parity = 0;
    for (int base = 0; base < N; base += kPaintThreads) {
      const int i = base + tid;
      int2 b = make_int2(kHidden, kHidden);
      if (i < N) b = fbox[i];
      const bool hit = b.x >= lo_x && b.x <= hi_x && b.y >= lo_y && b.y <= hi_y;
      const unsigned ballot = __ballot_sync(0xffffffffu, hit);
      if (lane == 0) warp_hits[parity][warp] = __popc(ballot);
      // One barrier per scan chunk: warp_hits is double-buffered, and the list is only refilled
      // after the barrier that ends a drain.
      __syncthreads();
      int before = 0, total = 0;
#pragma unroll
      for (int w = 0; w < kWarps; ++w) {
        const int c = warp_hits[parity][w];
        before += (w < warp) ? c : 0;
        total += c;
      }
      if (hit) {
        const double2 c = fcentre[i];
        const double x1 = (double)b.x, y1 = (double)b.y;
        PaintEntry e;
        e.wx1 = __dsub_rn(c.x, x1);
        e.wx2 = __dsub_rn(x1 + 1.0, c.x);
        e.wy1 = __dsub_rn(c.y, y1);
        e.wy2 = __dsub_rn(y1 + 1.0, c.y);
        e.x0 = b.x - r - 1;
        e.y0 = b.y - r - 1;
        const uint8_t* col = colors + (size_t)i * 3;
        e.rgb = (uint32_t)col[0] | ((uint32_t)col[1] << 8) | ((uint32_t)col[2] << 16);
        e.pad = 0;
        list[count + before + __popc(ballot & ((1u << lane) - 1u))] = e;
      }
      count += total;
      parity ^= 1;
      if (count <= kListCap - kPaintThreads && base + kPaintThreads < N) continue;

      __syncthreads();
      for (int n = 0; n < count; ++n) {
        const PaintEntry& e = list[n];
        const unsigned bc = (unsigned)px - (unsigned)e.x0;  // patch column
        if (bc > last) continue;
        const int ca = (int)bc - r - 1;  // icon column offset of the copies padded on the right
        const double qa = sq(ca), qb = sq(ca - 1);
        const double c0 = (double)(e.rgb & 0xff), c1 = (double)((e.rgb >> 8) & 0xff),
                     c2 = (double)(e.rgb >> 16);
#pragma unroll
        for (int k = 0; k < kRowsPerThread; ++k) {
          const unsigned br = (unsigned)py[k] - (unsigned)e.y0;  // patch row
          if (br > last) continue;
          const int ra = (int)br - r - 1;
          const double ya = sq(ra), yb = sq(ra - 1);
          // the four shifted copies: icon1 padded bottom / right, icon2 top / right, icon3
          // bottom / left, icon4 top / left
          const bool top = br >= 1, bottom = br < last, left = bc >= 1, right = bc < last;
          const double i1 = (bottom && right) ? icon_value(__dadd_rn(ya, qa), half_r2, scale) : 0.0;
          const double i2 = (top && right) ? icon_value(__dadd_rn(yb, qa), half_r2, scale) : 0.0;
          const double i3 = (bottom && left) ? icon_value(__dadd_rn(ya, qb), half_r2, scale) : 0.0;
          const double i4 = (top && left) ? icon_value(__dadd_rn(yb, qb), half_r2, scale) : 0.0;
          // ((icon1 wx2) wy2 + (icon2 wx2) wy1) + (icon3 wx1) wy2 + (icon4 wx1) wy1, left to right
          double p = __dmul_rn(__dmul_rn(i1, e.wx2), e.wy2);
          p = __dadd_rn(p, __dmul_rn(__dmul_rn(i2, e.wx2), e.wy1));
          p = __dadd_rn(p, __dmul_rn(__dmul_rn(i3, e.wx1), e.wy2));
          p = __dadd_rn(p, __dmul_rn(__dmul_rn(i4, e.wx1), e.wy1));
          if (p == 0.0) continue;  // (1 - 0) v + 0 c == v exactly
          const double keep = __dsub_rn(1.0, p);
          v[k][0] = trunc(__dadd_rn(__dmul_rn(keep, v[k][0]), __dmul_rn(p, c0)));
          v[k][1] = trunc(__dadd_rn(__dmul_rn(keep, v[k][1]), __dmul_rn(p, c1)));
          v[k][2] = trunc(__dadd_rn(__dmul_rn(keep, v[k][2]), __dmul_rn(p, c2)));
        }
      }
      __syncthreads();
      count = 0;
    }
  }

#pragma unroll
  for (int k = 0; k < kRowsPerThread; ++k) {
    if (py[k] < 0) continue;
    uint8_t* p = out + frame_off + ((size_t)py[k] * W + px) * 3;
    // the blend stays in [-1e-13, 255 + 1e-13]: truncation toward zero is numpy's uint8 cast
    p[0] = (uint8_t)__double2int_rz(v[k][0]);
    p[1] = (uint8_t)__double2int_rz(v[k][1]);
    p[2] = (uint8_t)__double2int_rz(v[k][2]);
  }
}

}  // namespace

int paint_radius(int H, int W) {
  // int(round(min(H, W) * 0.015)): float64 product, Python's round half to even (rint)
  return (int)std::rint((double)std::min(H, W) * 0.015);
}

size_t paint_point_track_workspace_bytes(long long frames, long long points) {
  if (frames <= 0 || points <= 0) return 0;
  const unsigned long long n = (unsigned long long)frames * (unsigned long long)points;
  if (n > (1ull << 56)) return SIZE_MAX;  // no allocation can hold it
  return align_up(n * sizeof(int2), 256) + n * sizeof(double2);
}

int paint_point_track(const uint8_t* frames, int T, int H, int W, const void* tracks, int tracks_fp64,
                      const uint8_t* visibles, int N, const uint8_t* colors, uint8_t* out,
                      void* ws, cudaStream_t s) {
  const int tiles_x = ceil_div(W, kTile), tiles_per_frame = tiles_x * ceil_div(H, kTile);
  const size_t n = (size_t)T * N;
  int2* box = static_cast<int2*>(ws);
  double2* centre = reinterpret_cast<double2*>(static_cast<char*>(ws) + align_up(n * sizeof(int2), 256));
  if (N > 0) {
    ProfileScope ps("paint_footprint", s, 0.0, (double)n * ((tracks_fp64 ? 16 : 8) + 1 + 24));
    const unsigned grid = (unsigned)std::min<long long>(ceil_div_ll((long long)n, 256), (long long)num_sms() * 16);
    if (tracks_fp64)
      paint_footprint_kernel<<<grid, 256, 0, s>>>(static_cast<const double*>(tracks), visibles, T, N, H, W,
                                                  box, centre);
    else
      paint_footprint_kernel<<<grid, 256, 0, s>>>(static_cast<const float*>(tracks), visibles, T, N, H, W,
                                                  box, centre);
    count_launch();
    TAPIR_LAUNCH_CHECK("paint_footprint_kernel");
  }
  ProfileScope ps("paint_tiles", s, 0.0, (double)T * H * W * 6 + (double)n * 24);
  paint_tiles_kernel<<<(unsigned)((long long)T * tiles_per_frame), kPaintThreads, 0, s>>>(
      frames, out, H, W, N, paint_radius(H, W), tiles_x, tiles_per_frame, box, centre, colors);
  count_launch();
  TAPIR_LAUNCH_CHECK("paint_tiles_kernel");
  return kOk;
}

}  // namespace tapir
