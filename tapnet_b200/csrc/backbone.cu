// Feature-pyramid backbone (SURVEY.md 8(a3)): ResNet-V2 + InstanceNorm, ExtraConvs, L2 norm.
// All 3x3 / 1x1 convolutions run as split-bf16 wgmma GEMMs (gemm_tc.cu); this file holds the
// HBM-bound kernels around them (stem conv, instance/layer norm, im2col for the three
// stride-2 layers, resize) and the per-frame-chunk orchestration.
#include "kernels.cuh"

namespace tapir {

namespace {

// ------------------------------------------------------------------------ split planes
__global__ void split_planes_kernel(const float* __restrict__ src, long long ld_src,
                                    __nv_bfloat16* __restrict__ dst, long long ld_dst,
                                    long long plane_stride, long long rows, int cols,
                                    int cols_padded, int planes) {
  const long long total = rows * cols_padded;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / cols_padded;
    const int c = (int)(i - r * cols_padded);
    float v = (c < cols) ? src[r * ld_src + c] : 0.f;
    for (int q = 0; q < planes; ++q) {
      __nv_bfloat16 h = __float2bfloat16_rn(v);
      v -= __bfloat162float(h);
      dst[q * plane_stride + r * ld_dst + c] = h;
    }
  }
}

// ------------------------------------------------------------------------ stem conv
// nets.py:395-402,420: F.pad(x,(2,4,2,4)) then 7x7 stride-2 conv, 3 -> 64, no bias.
// CTA = 16 x 32 output pixels; each thread owns two pixels of a row (16 apart) and all 64
// output channels (one broadcast LDS.128 of weights feeds 8 FMAs; with one pixel per thread the
// kernel was bound by the shared-memory pipe, not the FMA pipe).
constexpr int kStemTileY = 16;
constexpr int kStemTileX = 32;
constexpr int kStemPatchY = 2 * kStemTileY + 5;  // 37 input rows
constexpr int kStemPatchX = 2 * kStemTileX + 5;  // 69 input columns

// In = float: video already in [-1,1].  In = uint8_t: raw [0,255] frames, normalised on load
// exactly like preprocess_frames (pytorch_live_demo.py:30-41: x / 255 * 2 - 1, fp32, each
// operation rounded) so that the float tensor never exists in HBM (SURVEY 8f row 1).
__device__ __forceinline__ float stem_load(const float* p) { return *p; }
__device__ __forceinline__ float stem_load(const uint8_t* p) {
  return __fsub_rn(__fmul_rn(__fdiv_rn((float)*p, 255.f), 2.f), 1.f);
}

// Patch loaders: value of channel c at pixel (y, x) of frame f of the H x W input.
template <typename In>
struct StemRgb {
  static constexpr int kTableFloats = 0;
  const In* __restrict__ video;
  __device__ __forceinline__ void prepare(float*) const {}
  __device__ __forceinline__ float operator()(const float*, int f, int H, int W, int y, int x,
                                              int c) const {
    const In v = __ldg(video + (((long long)f * H + y) * W + x) * 3 + c);
    return stem_load(&v);
  }
};

// YUV (Reader = YuvReader<uint8_t> or YuvReader<uint16_t>): the integer conversion gives the
// uint8 RGB byte, and a per-CTA table of the 256 stem_load values gives exactly the float the
// uint8 loader computes from that byte.
template <typename Reader>
struct StemYuv {
  static constexpr int kTableFloats = 256;
  Reader src;
  __device__ __forceinline__ void prepare(float* table) const {
    for (int i = threadIdx.x; i < 256; i += blockDim.x) {
      const uint8_t b = (uint8_t)i;
      table[i] = stem_load(&b);
    }
    __syncthreads();
  }
  __device__ __forceinline__ float operator()(const float* table, int f, int, int, int y, int x,
                                              int c) const {
    uint8_t rgb[3];
    src.pixel(f, y, x, rgb);
    return table[c == 0 ? rgb[0] : (c == 1 ? rgb[1] : rgb[2])];
  }
};

template <typename Load>
__global__ void __launch_bounds__(256, 1) stem_conv_kernel(const Load load,
                                                           const float* __restrict__ w, int H, int W,
                                                           float* __restrict__ out) {
  extern __shared__ float stem_smem[];
  float* ws = stem_smem;                    // [147][64]
  float* patch = stem_smem + 147 * 64;      // [37][69][3]
  float* table = patch + kStemPatchY * kStemPatchX * 3;  // [Load::kTableFloats]
  const int OH = H / 2, OW = W / 2;
  const int f = blockIdx.z;
  const int oy0 = blockIdx.y * kStemTileY, ox0 = blockIdx.x * kStemTileX;
  for (int i = threadIdx.x; i < 147 * 64; i += 256) ws[i] = w[i];
  load.prepare(table);
  const int iy0 = 2 * oy0 - 2, ix0 = 2 * ox0 - 2;
  for (int i = threadIdx.x; i < kStemPatchY * kStemPatchX * 3; i += 256) {
    const int c = i % 3, px = (i / 3) % kStemPatchX, py = i / (3 * kStemPatchX);
    const int y = iy0 + py, x = ix0 + px;
    float v = 0.f;
    if (y >= 0 && y < H && x >= 0 && x < W) v = load(table, f, H, W, y, x, c);
    patch[i] = v;
  }
  __syncthreads();
  const int ty = threadIdx.x / 16, tx = threadIdx.x % 16;  // pixels (ty, tx) and (ty, tx + 16)
  float acc0[64], acc1[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) acc0[i] = acc1[i] = 0.f;
  for (int ky = 0; ky < 7; ++ky) {
    for (int kx = 0; kx < 7; ++kx) {
      const float* pp = patch + ((2 * ty + ky) * kStemPatchX + (2 * tx + kx)) * 3;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float v0 = pp[c], v1 = pp[c + 2 * 16 * 3];
        const float4* wr = reinterpret_cast<const float4*>(ws + ((ky * 7 + kx) * 3 + c) * 64);
#pragma unroll
        for (int o = 0; o < 16; ++o) {
          const float4 w4 = wr[o];
          acc0[4 * o + 0] = fmaf(v0, w4.x, acc0[4 * o + 0]);
          acc0[4 * o + 1] = fmaf(v0, w4.y, acc0[4 * o + 1]);
          acc0[4 * o + 2] = fmaf(v0, w4.z, acc0[4 * o + 2]);
          acc0[4 * o + 3] = fmaf(v0, w4.w, acc0[4 * o + 3]);
          acc1[4 * o + 0] = fmaf(v1, w4.x, acc1[4 * o + 0]);
          acc1[4 * o + 1] = fmaf(v1, w4.y, acc1[4 * o + 1]);
          acc1[4 * o + 2] = fmaf(v1, w4.z, acc1[4 * o + 2]);
          acc1[4 * o + 3] = fmaf(v1, w4.w, acc1[4 * o + 3]);
        }
      }
    }
  }
  const int oy = oy0 + ty;
  if (oy < OH) {
    if (ox0 + tx < OW) {
      float4* o = reinterpret_cast<float4*>(out + (((long long)f * OH + oy) * OW + ox0 + tx) * 64);
#pragma unroll
      for (int i = 0; i < 16; ++i) o[i] = make_float4(acc0[4 * i], acc0[4 * i + 1], acc0[4 * i + 2], acc0[4 * i + 3]);
    }
    if (ox0 + tx + 16 < OW) {
      float4* o = reinterpret_cast<float4*>(out + (((long long)f * OH + oy) * OW + ox0 + tx + 16) * 64);
#pragma unroll
      for (int i = 0; i < 16; ++i) o[i] = make_float4(acc1[4 * i], acc1[4 * i + 1], acc1[4 * i + 2], acc1[4 * i + 3]);
    }
  }
}

// ------------------------------------------------------------------------ instance norm
// nets.py:280-286: per (frame, channel) statistics over H*W, biased variance, eps 1e-5.
// Sums are accumulated in fp64 (sum, sum of squares) so E[x^2]-E[x]^2 is exact to fp32.
constexpr int kStatPixelsPerBlock = 1024;

__global__ void __launch_bounds__(256) instnorm_stats_kernel(const float* __restrict__ x,
                                                             long long hw, int C,
                                                             double* __restrict__ sums,
                                                             int pixels_per_block) {
  __shared__ double red[256 * 8];
  const int f = blockIdx.y;
  const int c4n = C / 4;             // float4 groups per pixel
  const int lanes = 256 / c4n;       // pixel lanes per block
  const int g = threadIdx.x % c4n, pl = threadIdx.x / c4n;
  const long long p0 = (long long)blockIdx.x * pixels_per_block;
  long long p1 = p0 + pixels_per_block;
  if (p1 > hw) p1 = hw;
  double s[4] = {0, 0, 0, 0}, ss[4] = {0, 0, 0, 0};
  if (pl < lanes) {
    const float4* base = reinterpret_cast<const float4*>(x + (long long)f * hw * C);
    for (long long p = p0 + pl; p < p1; p += lanes) {
      const float4 v = base[p * c4n + g];
      s[0] += v.x; ss[0] += (double)v.x * v.x;
      s[1] += v.y; ss[1] += (double)v.y * v.y;
      s[2] += v.z; ss[2] += (double)v.z * v.z;
      s[3] += v.w; ss[3] += (double)v.w * v.w;
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    red[threadIdx.x * 8 + i] = s[i];
    red[threadIdx.x * 8 + 4 + i] = ss[i];
  }
  __syncthreads();
  // thread t < C reduces channel t over the pixel lanes
  if (threadIdx.x < C) {
    const int c = threadIdx.x;
    const int gg = c / 4, e = c % 4;
    double a = 0, b = 0;
    for (int l = 0; l < lanes; ++l) {
      a += red[(l * c4n + gg) * 8 + e];
      b += red[(l * c4n + gg) * 8 + 4 + e];
    }
    atomicAdd(&sums[((long long)f * C + c) * 2 + 0], a);
    atomicAdd(&sums[((long long)f * C + c) * 2 + 1], b);
  }
}

// relu(x * scale + shift) -> bf16 planes.  CTA = one frame x a chunk of pixels; a thread keeps
// its 4 channels' (scale, shift) in registers and streams pixels, 4 independent loads in flight.
constexpr int kApplyPixelsPerBlock = 512;
// The statistics are finalised here, per thread, from the fp64 sums (scale = w / sqrt(var + eps),
// shift = b - mean * scale, in fp64): one launch instead of two per norm.  `zero_next` (nullable)
// is the OTHER statistics buffer of the ping-pong pair: the GEMM that follows accumulates into it,
// and the first pixel block of every frame clears that frame's entries here, which replaces a
// memset node per norm (31 fewer graph nodes per streaming frame in total).
__global__ void __launch_bounds__(256) instnorm_relu_split_kernel(
    const float* __restrict__ x, const double* __restrict__ sums, const float* __restrict__ w,
    const float* __restrict__ b, long long hw, int C, __nv_bfloat16* __restrict__ out,
    long long plane_stride, int planes, int pixels_per_block, double* __restrict__ zero_next,
    int zero_count) {
  const int f = blockIdx.y;
  const int c4n = C / 4;
  const int lanes = 256 / c4n;
  const int g = threadIdx.x % c4n, pl = threadIdx.x / c4n;
  float sc[4], sh[4];
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const int c = 4 * g + e;
    const long long i = (long long)f * C + c;
    const double mean = sums[2 * i] / (double)hw;
    double var = sums[2 * i + 1] / (double)hw - mean * mean;
    if (var < 0) var = 0;
    const double scale = (double)w[c] / sqrt(var + 1e-5);
    sc[e] = (float)scale;
    sh[e] = (float)((double)b[c] - mean * scale);
  }
  if (zero_next != nullptr && blockIdx.x == 0)
    for (int i = threadIdx.x; i < 2 * zero_count; i += 256) zero_next[(long long)f * 2 * zero_count + i] = 0.0;
  const long long p0 = (long long)blockIdx.x * pixels_per_block;
  long long p1 = p0 + pixels_per_block;
  if (p1 > hw) p1 = hw;
  const long long base = (long long)f * hw;
  const float4* xin = reinterpret_cast<const float4*>(x);
  for (long long p = p0 + pl; p < p1; p += 4 * lanes) {
    float4 v[4];
    long long idx[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const long long pp = p + (long long)u * lanes;
      idx[u] = (base + pp) * c4n + g;
      if (pp < p1) v[u] = xin[idx[u]];
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      if (p + (long long)u * lanes >= p1) continue;
      float y[4] = {fmaxf(fmaf(v[u].x, sc[0], sh[0]), 0.f), fmaxf(fmaf(v[u].y, sc[1], sh[1]), 0.f),
                    fmaxf(fmaf(v[u].z, sc[2], sh[2]), 0.f), fmaxf(fmaf(v[u].w, sc[3], sh[3]), 0.f)};
      for (int q = 0; q < planes; ++q) {
        uint2 pk;
        pk.x = bf16x2_split(y[0], y[1]);
        pk.y = bf16x2_split(y[2], y[3]);
        reinterpret_cast<uint2*>(out + q * plane_stride)[idx[u]] = pk;
      }
    }
  }
}

// ------------------------------------------------------------------------ im2col, stride 2
// nets.py:258-267,320: stride-2 3x3 convs see F.pad(x,(0,2,0,2)): tap (ky,kx) reads
// in[2y+ky, 2x+kx], zero beyond the border; the 1x1 stride-2 projection reads in[2y,2x].
__global__ void __launch_bounds__(256) im2col_s2_kernel(const __nv_bfloat16* __restrict__ in,
                                                        long long in_plane_stride, int H, int W,
                                                        int C, int taps,
                                                        __nv_bfloat16* __restrict__ out,
                                                        long long out_plane_stride, int planes,
                                                        long long total8) {
  const int OH = H / 2, OW = W / 2;
  const int c8n = C / 8;
  const int kside = (taps == 9) ? 3 : 1;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total8;
       i += (long long)gridDim.x * blockDim.x) {
    const int g = (int)(i % c8n);
    long long r = i / c8n;
    const int tap = (int)(r % taps);
    r /= taps;
    const int ox = (int)(r % OW);
    r /= OW;
    const int oy = (int)(r % OH);
    const long long f = r / OH;
    const int y = 2 * oy + tap / kside, x = 2 * ox + tap % kside;
    const bool ok = (y < H) && (x < W);
    const long long src = (((f * H + y) * W + x) * C) / 8 + g;
    for (int q = 0; q < planes; ++q) {
      uint4 v = make_uint4(0, 0, 0, 0);
      if (ok) v = reinterpret_cast<const uint4*>(in + q * in_plane_stride)[src];
      reinterpret_cast<uint4*>(out + q * out_plane_stride)[i] = v;
    }
  }
}

// ------------------------------------------------------------------------ layer norm
// nets.py:37-39,56 (affine+bias, channel-last) and nets.py:118-120,138-140 (scale only).
// One warp per row; C in {256, 512}.
template <int C>
__global__ void __launch_bounds__(256) layernorm_split_kernel(
    const float* __restrict__ x, long long rows, const float* __restrict__ w,
    const float* __restrict__ b, float* __restrict__ y, __nv_bfloat16* __restrict__ pl,
    long long plane_stride, int planes) {
  constexpr int V = C / 128;  // float4 per lane
  const int lane = threadIdx.x & 31;
  const long long row = blockIdx.x * (long long)(blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const float4* xr = reinterpret_cast<const float4*>(x + row * C);
  float4 v[V];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < V; ++i) {
    v[i] = xr[i * 32 + lane];
    s += v[i].x + v[i].y + v[i].z + v[i].w;
  }
  const float mean = warp_sum(s) * (1.0f / C);
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < V; ++i) {
    const float a = v[i].x - mean, bb = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
    ss += a * a + bb * bb + c * c + d * d;
  }
  const float rstd = 1.0f / sqrtf(warp_sum(ss) * (1.0f / C) + 1e-5f);
#pragma unroll
  for (int i = 0; i < V; ++i) {
    const int c0 = (i * 32 + lane) * 4;
    const float4 ww = reinterpret_cast<const float4*>(w)[i * 32 + lane];
    float o[4] = {(v[i].x - mean) * rstd * ww.x, (v[i].y - mean) * rstd * ww.y,
                  (v[i].z - mean) * rstd * ww.z, (v[i].w - mean) * rstd * ww.w};
    if (b != nullptr) {
      const float4 bb = reinterpret_cast<const float4*>(b)[i * 32 + lane];
      o[0] += bb.x; o[1] += bb.y; o[2] += bb.z; o[3] += bb.w;
    }
    if (y != nullptr) *reinterpret_cast<float4*>(y + row * C + c0) = make_float4(o[0], o[1], o[2], o[3]);
    if (pl != nullptr) {
      for (int q = 0; q < planes; ++q) {
        uint2 pk;
        pk.x = bf16x2_split(o[0], o[1]);
        pk.y = bf16x2_split(o[2], o[3]);
        *reinterpret_cast<uint2*>(pl + q * plane_stride + row * C + c0) = pk;
      }
    }
  }
}

// ------------------------------------------------------------------------ L2 normalise
// tapir_model.py:370-381: x / sqrt(max(sum x^2, 1e-12)) over channels.
template <int C>
__global__ void __launch_bounds__(256) l2norm_kernel(const float* __restrict__ x, long long rows,
                                                     float* __restrict__ out) {
  constexpr int V = C / 128;
  const int lane = threadIdx.x & 31;
  const long long row = blockIdx.x * (long long)(blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const float4* xr = reinterpret_cast<const float4*>(x + row * C);
  float4 v[V];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < V; ++i) {
    v[i] = xr[i * 32 + lane];
    s += v[i].x * v[i].x + v[i].y * v[i].y + v[i].z * v[i].z + v[i].w * v[i].w;
  }
  const float d = sqrtf(fmaxf(warp_sum(s), 1e-12f));
#pragma unroll
  for (int i = 0; i < V; ++i)
    reinterpret_cast<float4*>(out + row * C)[i * 32 + lane] =
        make_float4(v[i].x / d, v[i].y / d, v[i].z / d, v[i].w / d);
}

// ------------------------------------------------------------------------ bilinear resize
// utils.py:26-42 -> F.interpolate(mode='bilinear', align_corners=False), no antialias.
__global__ void __launch_bounds__(256) bilinear_resize_kernel(const float* __restrict__ src, int H,
                                                              int W, int C, float* __restrict__ dst,
                                                              int oH, int oW, long long total) {
  const float sy = (float)H / (float)oH, sx = (float)W / (float)oW;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    long long r = i / C;
    const int ox = (int)(r % oW);
    r /= oW;
    const int oy = (int)(r % oH);
    const long long f = r / oH;
    float fy = sy * (oy + 0.5f) - 0.5f;
    float fx = sx * (ox + 0.5f) - 0.5f;
    if (fy < 0.f) fy = 0.f;
    if (fx < 0.f) fx = 0.f;
    const int y0 = (int)fy, x0 = (int)fx;
    const int y1 = y0 + ((y0 < H - 1) ? 1 : 0), x1 = x0 + ((x0 < W - 1) ? 1 : 0);
    const float ly = fy - y0, lx = fx - x0;
    const float hy = 1.f - ly, hx = 1.f - lx;
    const float* b = src + f * (long long)H * W * C;
    const float v00 = b[((long long)y0 * W + x0) * C + c], v01 = b[((long long)y0 * W + x1) * C + c];
    const float v10 = b[((long long)y1 * W + x0) * C + c], v11 = b[((long long)y1 * W + x1) * C + c];
    dst[i] = hy * (hx * v00 + lx * v01) + ly * (hx * v10 + lx * v11);
  }
}

int grid_for(long long total, int block = 256) {
  long long g = ceil_div_ll(total, block);
  const long long cap = (long long)num_sms() * 16;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return (int)g;
}

}  // namespace

int split_planes(const float* src, long long ld_src, __nv_bfloat16* dst, long long ld_dst,
                 long long plane_stride, long long rows, int cols, int cols_padded, int planes,
                 cudaStream_t s) {
  TAPIR_CHECK_ARG(planes >= 1 && planes <= 3 && rows > 0 && cols > 0 && cols_padded >= cols &&
                      ld_dst >= cols_padded && ld_src >= cols,
                  "split_planes: bad shape rows=%lld cols=%d padded=%d", rows, cols, cols_padded);
  const long long total = rows * cols_padded;
  ProfileScope ps("split_planes", s, 0.0, (double)rows * cols * 4 + (double)total * 2 * planes);
  split_planes_kernel<<<grid_for(total), 256, 0, s>>>(src, ld_src, dst, ld_dst, plane_stride, rows,
                                                     cols, cols_padded, planes);
  count_launch();
  TAPIR_LAUNCH_CHECK("split_planes_kernel");
  return kOk;
}

template <typename Load>
int launch_stem_conv(const Load& load, const float* w_packed, int frames, int H, int W, float* out,
                     double input_bytes, cudaStream_t s) {
  TAPIR_CHECK_ARG(H % 2 == 0 && W % 2 == 0, "stem_conv: H, W must be even");
  const int smem = (147 * 64 + kStemPatchY * kStemPatchX * 3 + Load::kTableFloats) * (int)sizeof(float);
  static PerDeviceOnce configured;
  if (configured.pending()) {
    TAPIR_CUDA(cudaFuncSetAttribute(stem_conv_kernel<Load>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    configured.mark();
  }
  ProfileScope ps("backbone.stem_conv", s, 2.0 * frames * (H / 2) * (W / 2) * 64 * 147,
                  input_bytes + (double)frames * (H / 2) * (W / 2) * 64 * 4);
  dim3 grid(ceil_div(W / 2, kStemTileX), ceil_div(H / 2, kStemTileY), frames);
  stem_conv_kernel<Load><<<grid, 256, smem, s>>>(load, w_packed, H, W, out);
  count_launch();
  TAPIR_LAUNCH_CHECK("stem_conv_kernel");
  return kOk;
}

int stem_conv(const void* video, int video_u8, const float* w_packed, int frames, int H, int W,
              float* out, cudaStream_t s) {
  const double in_bytes = (double)frames * H * W * 3 * (video_u8 ? 1 : 4);
  if (video_u8)
    return launch_stem_conv(StemRgb<uint8_t>{static_cast<const uint8_t*>(video)}, w_packed, frames,
                            H, W, out, in_bytes, s);
  return launch_stem_conv(StemRgb<float>{static_cast<const float*>(video)}, w_packed, frames, H, W,
                          out, in_bytes, s);
}

int stem_conv_yuv(const tapir_yuv_frames& video, const float* w_packed, int frames, int H, int W,
                  float* out, cudaStream_t s) {
  const YuvLayout l = yuv_layout(video);
  const double in_bytes = frames * yuv_window_bytes(video);
  if (video.sample_bytes == 1)
    return launch_stem_conv(StemYuv<YuvReader<uint8_t>>{{l}}, w_packed, frames, H, W, out, in_bytes, s);
  return launch_stem_conv(StemYuv<YuvReader<uint16_t>>{{l}}, w_packed, frames, H, W, out, in_bytes, s);
}

int instnorm_stats(const float* x, int frames, long long hw, int C, double* sums, cudaStream_t s) {
  TAPIR_CHECK_ARG(C == 64 || C == 128 || C == 256, "instnorm_stats: C=%d unsupported", C);
  ProfileScope ps("backbone.instnorm_stats", s, 0.0, (double)frames * hw * C * 4);
  TAPIR_CUDA(cudaMemsetAsync(sums, 0, sizeof(double) * 2 * frames * C, s));
  // single frames (streaming): 1024-pixel blocks would be 16 CTAs; shrink until every SM has one
  int ppb = kStatPixelsPerBlock;
  while (ppb > 64 && ceil_div_ll(hw, ppb) * frames < (long long)num_sms()) ppb /= 2;
  dim3 grid((unsigned)ceil_div_ll(hw, ppb), frames);
  instnorm_stats_kernel<<<grid, 256, 0, s>>>(x, hw, C, sums, ppb);
  count_launch();
  TAPIR_LAUNCH_CHECK("instnorm_stats_kernel");
  return kOk;
}

int instnorm_relu_split(const float* x, const double* sums, const float* w, const float* b,
                        int frames, long long hw, int C, __nv_bfloat16* out, long long plane_stride,
                        int planes, double* zero_next, int zero_channels, cudaStream_t s) {
  const long long total4 = (long long)frames * hw * C / 4;
  ProfileScope ps("backbone.instnorm_apply", s, 0.0, (double)total4 * (16 + 8 * planes));
  // single frames (streaming): 512-pixel blocks would give 32 CTAs of 8 dependent load rounds
  // each; shrink the block until every SM has work (down to one load round per thread)
  int ppb = kApplyPixelsPerBlock;
  const int min_ppb = 4 * (256 / (C / 4));
  while (ppb > min_ppb && ceil_div_ll(hw, ppb) * frames < 2ll * num_sms()) ppb /= 2;
  dim3 grid((unsigned)ceil_div_ll(hw, ppb), frames);
  instnorm_relu_split_kernel<<<grid, 256, 0, s>>>(x, sums, w, b, hw, C, out, plane_stride, planes, ppb,
                                                  zero_next, zero_channels);
  count_launch();
  TAPIR_LAUNCH_CHECK("instnorm_relu_split_kernel");
  return kOk;
}

int im2col_s2(const __nv_bfloat16* in, long long in_plane_stride, int frames, int H, int W, int C,
              int taps, __nv_bfloat16* out, long long out_plane_stride, int planes, cudaStream_t s) {
  TAPIR_CHECK_ARG((taps == 1 || taps == 9) && C % 8 == 0 && H % 2 == 0 && W % 2 == 0,
                  "im2col_s2: bad arguments");
  const long long total8 = (long long)frames * (H / 2) * (W / 2) * taps * (C / 8);
  ProfileScope ps("backbone.im2col", s, 0.0, (double)total8 * 32 * planes);
  im2col_s2_kernel<<<grid_for(total8), 256, 0, s>>>(in, in_plane_stride, H, W, C, taps, out,
                                                   out_plane_stride, planes, total8);
  count_launch();
  TAPIR_LAUNCH_CHECK("im2col_s2_kernel");
  return kOk;
}

int layernorm_split(const float* x, long long rows, int C, const float* w, const float* b,
                    float* y, __nv_bfloat16* planes_out, long long plane_stride, int planes,
                    cudaStream_t s) {
  ProfileScope ps("layernorm", s, 0.0, (double)rows * C * (4 + (y ? 4 : 0) + (planes_out ? 2 * planes : 0)));
  const unsigned grid = (unsigned)ceil_div_ll(rows, 8);
  if (C == 256) {
    layernorm_split_kernel<256><<<grid, 256, 0, s>>>(x, rows, w, b, y, planes_out, plane_stride, planes);
  } else if (C == 512) {
    layernorm_split_kernel<512><<<grid, 256, 0, s>>>(x, rows, w, b, y, planes_out, plane_stride, planes);
  } else {
    set_error("layernorm_split: C=%d unsupported", C);
    return kUnsupported;
  }
  count_launch();
  TAPIR_LAUNCH_CHECK("layernorm_split_kernel");
  return kOk;
}

int l2_normalize(const float* x, long long rows, int C, float* out, cudaStream_t s) {
  ProfileScope ps("l2norm", s, 0.0, (double)rows * C * 8);
  const unsigned grid = (unsigned)ceil_div_ll(rows, 8);
  if (C == 128) {
    l2norm_kernel<128><<<grid, 256, 0, s>>>(x, rows, out);
  } else if (C == 256) {
    l2norm_kernel<256><<<grid, 256, 0, s>>>(x, rows, out);
  } else {
    set_error("l2_normalize: C=%d unsupported", C);
    return kUnsupported;
  }
  count_launch();
  TAPIR_LAUNCH_CHECK("l2norm_kernel");
  return kOk;
}

int bilinear_resize(const float* src, int frames, int H, int W, int C, float* dst, int oH, int oW,
                    cudaStream_t s) {
  const long long total = (long long)frames * oH * oW * C;
  ProfileScope ps("resize", s, 0.0, (double)total * 8);
  bilinear_resize_kernel<<<grid_for(total), 256, 0, s>>>(src, H, W, C, dst, oH, oW, total);
  count_launch();
  TAPIR_LAUNCH_CHECK("bilinear_resize_kernel");
  return kOk;
}

// ------------------------------------------------------------------------ orchestration

namespace {

constexpr size_t kBackboneSplitKBytes = 40u << 20;

struct BackbonePlan {
  float* buf[4];            // fp32 activation buffers (ping-pong / shortcut / conv_0 output)
  __nv_bfloat16* act;       // normalised activation planes
  __nv_bfloat16* col;       // im2col planes (stride-2 layers) / ExtraConvs hidden planes
  double* sums[2];          // instance-norm statistics (fp64 sum, sum of squares), ping-pong:
                            // a norm reads one while the next GEMM's epilogue fills the other
  float* splitk;            // split-K scratch for single-frame (streaming) calls
  long long act_plane, col_plane;
};

size_t plan_backbone(Arena& a, int frames, int H, int W, int extra, int planes, BackbonePlan* bp) {
  const long long px = (long long)frames * H * W;
  const long long act_elems = px / 4 * 64;  // largest activation: [F, H/2, W/2, 64] == 16*px
  for (int i = 0; i < 4; ++i) bp->buf[i] = a.take<float>(act_elems);
  bp->act_plane = act_elems;
  bp->act = a.take<__nv_bfloat16>(act_elems * planes);
  // im2col of group-1 conv_0: [F*H/4*W/4, 9*64]; ExtraConvs hidden: [F*H/8*W/8, 1024]
  long long col_elems = px / 16 * 576;
  const long long hid = px / 64 * 1024;
  if (extra && hid > col_elems) col_elems = hid;
  bp->col_plane = col_elems;
  bp->col = a.take<__nv_bfloat16>(col_elems * planes);
  bp->sums[0] = a.take<double>((size_t)frames * 256 * 2);
  bp->sums[1] = a.take<double>((size_t)frames * 256 * 2);
  bp->splitk = a.take<float>(kBackboneSplitKBytes / sizeof(float));
  return a.off;
}

// An ExtraConv GEMM: split-K only for single-frame (streaming) passes, see GemmArgs::allow_splitk.
GemmArgs extra_conv_args(const tapir_linear& l, const BackbonePlan& bp, int frames) {
  GemmArgs g = gemm_args(l);
  g.splitk_ws = bp.splitk; g.splitk_ws_bytes = kBackboneSplitKBytes; g.allow_splitk = (frames == 1);
  return g;
}

}  // namespace

size_t backbone_workspace_bytes(int frames, int H, int W, int extra_convs, int planes) {
  Arena a(nullptr, 0);
  BackbonePlan bp;
  return plan_backbone(a, frames, H, W, extra_convs, planes, &bp) + 256;
}

int backbone_stem(const tapir_backbone_weights* w, const void* video_chunk, int video_u8,
                  int pass_frames, int H, int W, int frame0, int nframes, void* ws, size_t ws_bytes,
                  cudaStream_t s) {
  TAPIR_CHECK_ARG(w != nullptr && video_chunk != nullptr, "backbone_stem: null pointer");
  TAPIR_CHECK_ARG(pass_frames > 0 && frame0 >= 0 && nframes > 0 && frame0 + nframes <= pass_frames &&
                      H % 8 == 0 && W % 8 == 0 && H >= 16 && W >= 16,
                  "backbone_stem: bad frame range %d+%d of %d (H=%d W=%d)", frame0, nframes, pass_frames, H, W);
  Arena arena(ws, ws_bytes);
  BackbonePlan bp;
  plan_backbone(arena, pass_frames, H, W, w->num_extra > 0, w->planes, &bp);
  if (!arena.ok) {
    set_error("backbone_stem: workspace too small (%zu < %zu)", ws_bytes, arena.off);
    return kWorkspaceTooSmall;
  }
  float* out = bp.buf[0] + (size_t)frame0 * (H / 2) * (W / 2) * 64;
  return stem_conv(video_chunk, video_u8, w->stem_w, nframes, H, W, out, s);
}

int backbone_forward(const tapir_backbone_weights* w, const void* video, int video_u8, int frames,
                     int H, int W, float* lowres, float* hires, void* ws, size_t ws_bytes,
                     cudaStream_t s, cudaEvent_t hires_ready, const tapir_yuv_frames* yuv) {
  // video == nullptr and yuv == nullptr: the stem output of all `frames` frames is already in
  // the workspace (tapir_backbone_stem, called per frame chunk while later chunks are still in
  // flight on PCIe).  yuv != nullptr: the stem reads the H x W window of YUV frames.
  TAPIR_CHECK_ARG(w != nullptr && lowres != nullptr && hires != nullptr, "backbone_forward: null pointer");
  TAPIR_CHECK_ARG(frames > 0 && H % 8 == 0 && W % 8 == 0 && H >= 16 && W >= 16,
                  "backbone_forward: image resolution must be a multiple of 8 (H=%d W=%d)", H, W);
  const int P = w->planes;
  TAPIR_CHECK_ARG(P >= 1 && P <= 3, "backbone_forward: planes=%d", P);
  Arena arena(ws, ws_bytes);
  BackbonePlan bp;
  plan_backbone(arena, frames, H, W, w->num_extra > 0, P, &bp);
  if (!arena.ok) {
    set_error("backbone_forward: workspace too small (%zu < %zu)", ws_bytes, arena.off);
    return kWorkspaceTooSmall;
  }

  int h = H / 2, wd = W / 2;
  float* x = bp.buf[0];
  if (yuv != nullptr)
    TAPIR_RETURN_IF(stem_conv_yuv(*yuv, w->stem_w, frames, H, W, x, s));
  else if (video != nullptr)
    TAPIR_RETURN_IF(stem_conv(video, video_u8, w->stem_w, frames, H, W, x, s));
  int xi = 0;  // index of the buffer holding x
  // InstanceNorm statistics are accumulated by the epilogue of the GEMM that produces the
  // tensor (fp64 atomics into bp.sums[.]); only the stem output needs the stand-alone pass.  The
  // two statistics buffers alternate: the norm kernel that reads one clears the other for the
  // GEMM that follows it.  sums[cur] = statistics of x.
  bool x_stats_ready = false;
  const int cur = 0;
  for (int bi = 0; bi < TAPIR_NUM_RESNET_BLOCKS; ++bi) {
    const tapir_resnet_block& b = w->blocks[bi];
    const long long m_in = (long long)frames * h * wd;
    const int oh = h / b.stride, ow = wd / b.stride;
    const long long m_out = (long long)frames * oh * ow;
    float* xnew = bp.buf[(xi + 1) & 3];
    float* shortcut_buf = bp.buf[(xi + 2) & 3];
    float* hbuf = bp.buf[(xi + 3) & 3];
    // bn_0 + relu -> planes
    if (!x_stats_ready) TAPIR_RETURN_IF(instnorm_stats(x, frames, (long long)h * wd, b.cin, bp.sums[cur], s));
    const bool fuse = (b.stride == 1) || (((long long)oh * ow) % 128 == 0);
    TAPIR_RETURN_IF(instnorm_relu_split(x, bp.sums[cur], b.bn0_w, b.bn0_b, frames, (long long)h * wd, b.cin,
                                        bp.act, bp.act_plane, P, fuse ? bp.sums[cur ^ 1] : nullptr, b.cout, s));
    const float* shortcut = x;
    if (b.has_proj) {
      GemmArgs g = gemm_args(b.proj);
      g.tag = "backbone.proj";
      g.M = (int)m_out;
      g.out_f32 = shortcut_buf;
      g.ldo = b.cout;
      if (b.stride == 1) {
        g.a = bp.act; g.lda = b.cin; g.a_plane_stride = bp.act_plane;
      } else {
        TAPIR_RETURN_IF(im2col_s2(bp.act, bp.act_plane, frames, h, wd, b.cin, 1, bp.col, bp.col_plane, P, s));
        g.a = bp.col; g.lda = b.cin; g.a_plane_stride = bp.col_plane;
      }
      TAPIR_RETURN_IF(gemm(g, s));
      shortcut = shortcut_buf;
    }
    {
      GemmArgs g = gemm_args(b.conv0);
      g.tag = "backbone.conv";
      g.M = (int)m_out;
      g.out_f32 = hbuf;
      g.ldo = b.cout;
      if (b.stride == 1) {
        g.mode = kGemmConv3x3;
        g.a = bp.act; g.a_plane_stride = bp.act_plane;
        g.frames = frames; g.H = h; g.W = wd; g.C = b.cin;
      } else {
        TAPIR_RETURN_IF(im2col_s2(bp.act, bp.act_plane, frames, h, wd, b.cin, 9, bp.col, bp.col_plane, P, s));
        g.a = bp.col; g.lda = 9 * b.cin; g.a_plane_stride = bp.col_plane;
      }
      if (fuse) {
        g.stats = bp.sums[cur ^ 1];  // cleared by the bn_0 norm kernel above
        g.rows_per_frame = oh * ow;
      }
      TAPIR_RETURN_IF(gemm(g, s));
      if (!fuse) TAPIR_RETURN_IF(instnorm_stats(hbuf, frames, (long long)oh * ow, b.cout, bp.sums[cur ^ 1], s));
    }
    const bool next_stats = (bi + 1 < TAPIR_NUM_RESNET_BLOCKS);  // statistics for the next block's bn_0
    TAPIR_RETURN_IF(instnorm_relu_split(hbuf, bp.sums[cur ^ 1], b.bn1_w, b.bn1_b, frames, (long long)oh * ow,
                                        b.cout, bp.act, bp.act_plane, P, next_stats ? bp.sums[cur] : nullptr,
                                        b.cout, s));
    {
      GemmArgs g = gemm_args(b.conv1);
      g.tag = "backbone.conv";
      g.mode = kGemmConv3x3;
      g.M = (int)m_out;
      g.a = bp.act; g.a_plane_stride = bp.act_plane;
      g.frames = frames; g.H = oh; g.W = ow; g.C = b.cout;
      g.residual = shortcut; g.ldr = b.cout;
      g.out_f32 = xnew; g.ldo = b.cout;
      x_stats_ready = next_stats;
      if (next_stats) g.stats = bp.sums[cur];  // cleared by the bn_1 norm kernel above
      TAPIR_RETURN_IF(gemm(g, s));
    }
    x = xnew;
    xi = (xi + 1) & 3;
    h = oh;
    wd = ow;
    (void)m_in;
    if (bi == 3) {  // resnet_unit_1 -> hires (tapir_model.py:356,376-381)
      TAPIR_RETURN_IF(l2_normalize(x, m_out, b.cout, hires, s));
      if (hires_ready != nullptr) TAPIR_CUDA(cudaEventRecord(hires_ready, s));
    }
  }
  const long long m = (long long)frames * h * wd;
  for (int e = 0; e < w->num_extra; ++e) {
    const tapir_extra_block& b = w->extra[e];
    float* y = bp.buf[(xi + 1) & 3];
    float* xnew = bp.buf[(xi + 2) & 3];
    TAPIR_RETURN_IF(layernorm_split(x, m, 256, b.ln_w, b.ln_b, y, bp.act, bp.act_plane, P, s));
    {
      GemmArgs g = extra_conv_args(b.conv, bp, frames);
      g.tag = "backbone.extra_conv";
      g.mode = kGemmConv3x3;
      g.M = (int)m;
      g.a = bp.act; g.a_plane_stride = bp.act_plane;
      g.frames = frames; g.H = h; g.W = wd; g.C = 256;
      g.act = 1;
      g.out_planes = bp.col; g.ldp = b.conv.N; g.out_plane_stride = bp.col_plane; g.out_P = P;
      TAPIR_RETURN_IF(gemm(g, s));
    }
    {
      GemmArgs g = extra_conv_args(b.conv1, bp, frames);
      g.tag = "backbone.extra_conv";
      g.mode = kGemmConv3x3;
      g.M = (int)m;
      g.a = bp.col; g.a_plane_stride = bp.col_plane;
      g.frames = frames; g.H = h; g.W = wd; g.C = b.conv.N;
      g.residual = y; g.ldr = 256;
      g.out_f32 = xnew; g.ldo = 256;
      TAPIR_RETURN_IF(gemm(g, s));
    }
    x = xnew;
    xi = (xi + 2) & 3;
  }
  TAPIR_RETURN_IF(l2_normalize(x, m, 256, lowres, s));
  return kOk;
}

}  // namespace tapir
