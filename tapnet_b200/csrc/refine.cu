// Refinement loop kernels (SURVEY.md 8(a7)-(a9)): pyramid pooling, fused bilinear-sample +
// dot local correlation (which also assembles the mixer input row), the depthwise-conv half
// of each PIPs mixer block, the mixer orchestration around the wgmma GEMMs, and the
// residual update.
#include "kernels.cuh"
#include "ptx.cuh"

namespace tapir {

namespace {

// ------------------------------------------------------------------------ a9 pooling
// tapir_model.py:519-527 avg_pool3d(kernel (2,2,1)) on [T,h,w,C] -> [T,h/2,w/2,C].
__global__ void __launch_bounds__(256) pool_kernel(const float4* __restrict__ in, int h, int w,
                                                   int c4n, float4* __restrict__ out,
                                                   long long total) {
  const int oh = h / 2, ow = w / 2;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int g = (int)(i % c4n);
    long long r = i / c4n;
    const int ox = (int)(r % ow);
    r /= ow;
    const int oy = (int)(r % oh);
    const long long t = r / oh;
    const long long base = ((t * h + 2 * oy) * w + 2 * ox) * c4n + g;
    const float4 a = in[base], b = in[base + c4n], c = in[base + (long long)w * c4n],
                 d = in[base + (long long)w * c4n + c4n];
    out[i] = make_float4((((a.x + b.x) + c.x) + d.x) * 0.25f, (((a.y + b.y) + c.y) + d.y) * 0.25f,
                         (((a.z + b.z) + c.z) + d.z) * 0.25f, (((a.w + b.w) + c.w) + d.w) * 0.25f);
  }
}

// ------------------------------------------------------------------------ a7 local correlation
// tapir_model.py:599-658 + utils.py:76-113.  For every (query n, frame t) and pyramid level:
//   c = pos * (gw, gh) / (init_w, init_h)              (grid coordinates, x then y)
//   49 samples at (y + dy, x + dx), dy, dx in -3..3, bilinear, zeros padding, where
//   grid_sample sees g = 2*(c / gh) - 1 for BOTH axes (the reference divides x by h too), so
//   the sampled pixel is  iy = ((2*(cy/gh)-1 + 1)*gh - 1)/2,  ix = ((2*(cx/gh)-1 + 1)*gw - 1)/2.
//   corr[s] = <bilinear patch feature, query feature>.
// Because the dot product is linear, we first dot every CELL of the bounding box of the 49
// samples with the query (one coalesced C-vector load per cell, 8 rows x <=16 columns), then
// combine 4 cell dots per sample with its bilinear weights: 64*C MACs instead of 196*C.
// One warp per level; the CTA (one (n,t) row) then writes the whole mixer input row
// [0, 0, occ, expd, feat(384), corr(49*L), 0-pad] as bf16 planes.
constexpr int kBoxRows = 8;
constexpr int kBoxColsMax = 16;
constexpr int kBoxCells = kBoxRows * kBoxColsMax;

struct CorrParams {
  tapir_corr_args a;
  int batch;  // clips; query q = b * a.num_points + n reads frame b * T + t of every level
  const int32_t* query_clip;  // or: a.num_points queries in all, query q of clip query_clip[q]
};

template <int V>  // V = C / 128 float4 per lane
__device__ __forceinline__ void cell_dots(const float* __restrict__ frame, int gh, int gw, int y0,
                                          int x0, int box_w, const float4 (&q)[V],
                                          float* __restrict__ table, int lane) {
  // cells are processed in groups of 32 (box index b = row * box_w + col)
  const int C = V * 128;
  const int ncell = kBoxRows * box_w;
  for (int b0 = 0; b0 < ncell; b0 += 32) {
    float part[32];
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      const int b = b0 + j;
      const int r = b / box_w, c = b - r * box_w;
      const int y = y0 + r, x = x0 + c;
      float acc = 0.f;
      if (b < ncell && y >= 0 && y < gh && x >= 0 && x < gw) {
        const float4* cp = reinterpret_cast<const float4*>(frame + ((long long)y * gw + x) * C);
#pragma unroll
        for (int v = 0; v < V; ++v) {
          const float4 f = __ldg(cp + v * 32 + lane);
          acc = fmaf(f.x, q[v].x, acc);
          acc = fmaf(f.y, q[v].y, acc);
          acc = fmaf(f.z, q[v].z, acc);
          acc = fmaf(f.w, q[v].w, acc);
        }
      }
      part[j] = acc;
    }
    // transpose-reduce: afterwards lane l holds the full dot product of cell b0 + l
#pragma unroll
    for (int s = 16; s >= 1; s >>= 1) {
#pragma unroll
      for (int j = 0; j < s; ++j) {
        const bool up = (lane & s) != 0;
        const float send = up ? part[j] : part[j + s];
        const float keep = up ? part[j + s] : part[j];
        part[j] = keep + __shfl_xor_sync(0xffffffffu, send, s);
      }
    }
    if (b0 + lane < kBoxCells) table[b0 + lane] = part[0];
  }
}

__global__ void __launch_bounds__(32 * TAPIR_MAX_CORR_LEVELS) local_corr_kernel(const CorrParams p) {
  __shared__ float table[TAPIR_MAX_CORR_LEVELS][kBoxCells];
  __shared__ float corr[TAPIR_MAX_CORR_LEVELS * 49];
  const tapir_corr_args& a = p.a;
  const int T = a.num_frames;
  // CTAs are issued frame-major: the CTAs resident at any time read the grids of one or two
  // frames (3.3 MB per frame at 256^2), which therefore stay in L2; the row order (n, t) of the
  // inputs / outputs would cycle through every frame's grids (all of them exceed L2) per query.
  // n is the query flattened over the clips, b its clip.
  const unsigned nq = (unsigned)a.num_points * (p.query_clip != nullptr ? 1u : (unsigned)p.batch);
  const int t = (int)(blockIdx.x / nq);
  const int n = (int)(blockIdx.x - (unsigned)t * nq);
  const int b = p.query_clip != nullptr ? p.query_clip[n] : n / a.num_points;
  const long long row = (long long)n * T + t;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const float px = a.pos[row * 2 + 0], py = a.pos[row * 2 + 1];
  const float* fhi = a.feat_hi + n * a.feat_hi_stride_n + t * a.feat_hi_stride_t;
  const float* flo = a.feat_lo + n * a.feat_lo_stride_n + t * a.feat_lo_stride_t;

  if (warp < a.num_levels) {
    const tapir_corr_level& L = a.levels[warp];
    const int gh = L.h, gw = L.w;
    // utils.convert_grid_coordinates (coords * out / in), tapir_model.py:603-606
    const float cx = __fdiv_rn(__fmul_rn(px, (float)gw), (float)a.init_w);
    const float cy = __fdiv_rn(__fmul_rn(py, (float)gh), (float)a.init_h);
    // pixel-space sample position of offset d:  ((2*((c+d)/gh) - 1 + 1) * size - 1) / 2
    auto pix = [&](float c, int d, int size) {
      const float g = __fsub_rn(__fmul_rn(2.f, __fdiv_rn(__fadd_rn(c, (float)d), (float)gh)), 1.f);
      return __fdiv_rn(__fsub_rn(__fmul_rn(__fadd_rn(g, 1.f), (float)size), 1.f), 2.f);
    };
    const int y0 = (int)floorf(pix(cy, -3, gh));
    const int x0 = (int)floorf(pix(cx, -3, gw));
    const int x_last = (int)floorf(pix(cx, 3, gw)) + 1;
    int box_w = x_last - x0 + 1;
    if (box_w < 2) box_w = 2;
    const float* frame = L.grid + ((long long)b * T + t) * gh * gw * L.C;
    if (box_w > kBoxColsMax) {
      // Wide grids (w/h > 2: the reference spaces the 49 samples gw/gh cells apart in x because it
      // normalises x by h, utils.py:104): the samples' cells no longer fit the 8 x 16 box, so
      // every sample is taken directly - 4 corner dot products each.  Same arithmetic, slower;
      // only panoramic aspect ratios come here.
      float4 q[2];
      const int V = L.C / 128;
      const float* qsrc = (L.C == 128) ? fhi : flo;
      q[0] = reinterpret_cast<const float4*>(qsrc)[lane];
      q[1] = (V == 2) ? reinterpret_cast<const float4*>(qsrc)[32 + lane] : make_float4(0, 0, 0, 0);
      for (int sidx = 0; sidx < 49; ++sidx) {
        const int dy = sidx / 7 - 3, dx = sidx % 7 - 3;
        const float iy = pix(cy, dy, gh), ix = pix(cx, dx, gw);
        const float fy0 = floorf(iy), fx0 = floorf(ix);
        const float wy1 = iy - fy0, wy0 = (fy0 + 1.f) - iy;
        const float wx1 = ix - fx0, wx0 = (fx0 + 1.f) - ix;
        float v = 0.f;
#pragma unroll
        for (int cr = 0; cr < 4; ++cr) {
          const int yy = (int)fy0 + (cr >> 1), xx = (int)fx0 + (cr & 1);
          float acc = 0.f;
          if (yy >= 0 && yy < gh && xx >= 0 && xx < gw) {
            const float4* cp = reinterpret_cast<const float4*>(frame + ((long long)yy * gw + xx) * L.C);
            for (int vv = 0; vv < V; ++vv) {
              const float4 f = __ldg(cp + vv * 32 + lane);
              acc = fmaf(f.x, q[vv].x, acc);
              acc = fmaf(f.y, q[vv].y, acc);
              acc = fmaf(f.z, q[vv].z, acc);
              acc = fmaf(f.w, q[vv].w, acc);
            }
          }
          acc = warp_sum(acc);
          v += acc * (((cr & 1) ? wx1 : wx0) * ((cr >> 1) ? wy1 : wy0));
        }
        if (lane == 0) corr[warp * 49 + sidx] = v;
      }
    } else {
    if (L.C == 128) {
      float4 q[1];
      q[0] = reinterpret_cast<const float4*>(fhi)[lane];
      cell_dots<1>(frame, gh, gw, y0, x0, box_w, q, table[warp], lane);
    } else {
      float4 q[2];
      q[0] = reinterpret_cast<const float4*>(flo)[lane];
      q[1] = reinterpret_cast<const float4*>(flo)[32 + lane];
      cell_dots<2>(frame, gh, gw, y0, x0, box_w, q, table[warp], lane);
    }
    __syncwarp();
    for (int sidx = lane; sidx < 49; sidx += 32) {
      const int dy = sidx / 7 - 3, dx = sidx % 7 - 3;
      const float iy = pix(cy, dy, gh), ix = pix(cx, dx, gw);
      const float fy0 = floorf(iy), fx0 = floorf(ix);
      const int ry = (int)fy0 - y0, rx = (int)fx0 - x0;
      // ATen grid_sampler bilinear weights
      const float wy1 = iy - fy0, wy0 = (fy0 + 1.f) - iy;
      const float wx1 = ix - fx0, wx0 = (fx0 + 1.f) - ix;
      // a corner can fall outside the box only through fp jitter at an exactly-integer
      // sample position, where its weight is ~1e-7: treating it as 0 is exact to fp32 noise
      const float* tb = table[warp];
      auto cell = [&](int r, int c) {
        return (r >= 0 && r < kBoxRows && c >= 0 && c < box_w) ? tb[r * box_w + c] : 0.f;
      };
      const float v = cell(ry, rx) * (wx0 * wy0) + cell(ry, rx + 1) * (wx1 * wy0) +
                      cell(ry + 1, rx) * (wx0 * wy1) + cell(ry + 1, rx + 1) * (wx1 * wy1);
      corr[warp * 49 + sidx] = v;
    }
    }  // box fits
  }
  __syncthreads();

  // ---- assemble the mixer input row (tapir_model.py:647-658), split into bf16 planes
  const int ncorr = 49 * a.num_levels;
  const float occ = a.occ[row], expd = a.expd[row];
  __nv_bfloat16* out = static_cast<__nv_bfloat16*>(a.out_planes);
  auto value = [&](int e) -> float {
    if (e < 2) return 0.f;  // position slots are zeroed (tapir_model.py:647)
    if (e == 2) return occ;
    if (e == 3) return expd;
    if (e < 4 + 128) return fhi[e - 4];
    if (e < 4 + 384) return flo[e - 132];
    if (e < 388 + ncorr) return corr[e - 388];
    return 0.f;
  };
  for (int e2 = threadIdx.x; e2 < a.ld / 2; e2 += blockDim.x) {
    float v0 = value(2 * e2), v1 = value(2 * e2 + 1);
    for (int q = 0; q < a.planes; ++q)
      *reinterpret_cast<uint32_t*>(out + q * a.out_plane_stride + row * a.ld + 2 * e2) = bf16x2_split(v0, v1);
  }
}

// ------------------------------------------------------------------------ a8 depthwise half
// nets.py:143-181 for one PIPsConvBlock, everything before the channel MLP:
//   y  = LN(x) * w                                   (scale only, eps 1e-5)
//   h1 = gelu(dwconv_k3(y; 512 -> 2048, 4 per channel) + b1)
//   h2 = dwconv_k3(h1; 2048) + b2 ;  z = x + sum of the 4 multipliers
//   out: z (fp32) and LN_1(z) * w1 as bf16 planes (the A operand of the `up` GEMM).
// Non-causal convs zero-pad one frame each side; causal convs look 2 frames back, with
// the optional context (last 2 frames of y and of h1 from the previous call) standing in for
// frames -2, -1 (nets.py:149-176).  CTA = QB queries x TT output frames (QB > 1 only for short clips /
// streaming, so that a CTA always has ~24 rows of work); thread = one of the 512 channels.
constexpr int kDwTileMax = 24;        // output frames per CTA (per query)
constexpr int kDwHalo = 4;            // extra layer-normed rows a tile needs (2+2 or 4+0)
constexpr int kDwRowBudget = 52;      // QB * (2*TT + 4) rows of 2 KB <= 104 KB (2 CTAs per SM)
constexpr int kDwSmallQueries = 8;    // max queries per CTA of the SMALL variant
constexpr int kDwCtxWindow = 4;       // of which this many have their hidden-state context in registers

struct DwParams {
  const float* x;
  float* z;
  __nv_bfloat16* planes_out;
  long long plane_stride;
  int planes;
  int T;
  int N;    // queries
  int TT;   // output frames per tile
  int QB;   // queries per CTA (short clips / streaming: several queries share one CTA)
  const float* ln_w;
  const float* w1;
  const float* b1;
  const float* w2;
  const float* b2;
  const float* ln1_w;
  const float* ctx1_in;
  const float* ctx2_in;
  float* ctx1_out;
  float* ctx2_out;
};

// One warp: LayerNorm (scale only, eps 1e-5) of a 512-wide row held as 4 float4 per lane.
__device__ __forceinline__ void ln512(const float4 (&v)[4], const float* __restrict__ w, int lane,
                                      float4 (&o)[4]) {
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) s += v[i].x + v[i].y + v[i].z + v[i].w;
  const float mean = warp_sum(s) * (1.0f / 512);
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
    ss += a * a + b * b + c * c + d * d;
  }
  const float rstd = 1.0f / sqrtf(warp_sum(ss) * (1.0f / 512) + 1e-5f);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float4 ww = reinterpret_cast<const float4*>(w)[i * 32 + lane];
    o[i] = make_float4((v[i].x - mean) * rstd * ww.x, (v[i].y - mean) * rstd * ww.y,
                       (v[i].z - mean) * rstd * ww.z, (v[i].w - mean) * rstd * ww.w);
  }
}

// SMALL = several queries per CTA (short clips / streaming): one CTA per SM, 128 registers, and
// the causal hidden-state context of the next query is prefetched into registers.
template <bool CAUSAL, bool SMALL>
__global__ void __launch_bounds__(512, SMALL ? 1 : 2) mixer_dw_kernel(const DwParams p) {
  extern __shared__ float dw_smem[];
  const int TT = p.TT, QB = p.QB, T = p.T;
  const int RY = TT + kDwHalo;              // layer-normed rows per query
  float* ybuf = dw_smem;                    // [QB][RY][512]  (rows are recycled for z)
  float* xraw = dw_smem + QB * RY * 512;    // [QB][TT][512]  raw rows for the skip connection
  const int t0 = blockIdx.x * TT;
  const int t1 = min(t0 + TT, T);
  const int n0 = blockIdx.y * QB;
  const int nq = min(QB, p.N - n0);
  const int c = threadIdx.x;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // smem row r of a query <-> frame lo + r: non-causal needs t0-2 .. t1+1, causal t0-4 .. t1-1
  const int lo = CAUSAL ? t0 - 4 : t0 - 2;
  const int nrow = (CAUSAL ? t1 : t1 + 2) - lo;

  // Causal context of the hidden activation (frames -2, -1 of h1; only the first tile of a clip
  // reads it).  With several queries per CTA (short clips, streaming) these were three dependent
  // global loads per query, serialised over the queries (8 x 3 x ~0.7 us of a 23 us launch at
  // T = 1); the SMALL variant issues all of them up front, before phase 1, so that the 16 KB per
  // query stream in while the rows are layer-normed (the launch moves 46 MB of context at 1024
  // points: it is bandwidth bound once the loads overlap).
  const bool has_ctx2 = CAUSAL && p.ctx2_in != nullptr && t0 == 0;
  // rolling window: the context of queries q .. q + 3 is in flight / in registers; slot q % 4 is
  // refilled with query q + 4 as soon as query q has consumed it
  float4 ctx_all[SMALL ? kDwCtxWindow : 1][2];
  auto fetch_ctx2 = [&](int q, float4 (&dst)[2]) {
    dst[0] = dst[1] = make_float4(0, 0, 0, 0);
    if (has_ctx2 && q < nq) {
      const float* src = p.ctx2_in + ((long long)(n0 + q) * 2) * 2048 + 4 * c;
      dst[0] = *reinterpret_cast<const float4*>(src);
      dst[1] = *reinterpret_cast<const float4*>(src + 2048);
    }
  };
  if (SMALL) {
#pragma unroll
    for (int q = 0; q < kDwCtxWindow; ++q) fetch_ctx2(q, ctx_all[q]);
  }

  // ---- phase 1: y = LN(x) * w for every needed row (one warp per row)
  for (int rq = warp; rq < nq * nrow; rq += 16) {
    const int q = rq / nrow, r = rq - q * nrow;
    const int t = lo + r, n = n0 + q;
    float4* dst = reinterpret_cast<float4*>(ybuf + (q * RY + r) * 512);
    if (t >= 0 && t < T) {
      const float4* xr = reinterpret_cast<const float4*>(p.x + ((long long)n * T + t) * 512);
      float4 v[4], o[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) v[i] = xr[i * 32 + lane];
      ln512(v, p.ln_w, lane, o);
#pragma unroll
      for (int i = 0; i < 4; ++i) dst[i * 32 + lane] = o[i];
      if (t >= t0 && t < t1) {  // the frame loop below must not wait on L2 for the skip input
        float4* xd = reinterpret_cast<float4*>(xraw + (q * TT + (t - t0)) * 512);
#pragma unroll
        for (int i = 0; i < 4; ++i) xd[i * 32 + lane] = v[i];
      }
    } else if (CAUSAL && p.ctx1_in != nullptr && t >= -2 && t < 0) {
      // context frames -2, -1 of the layer-normed input (nets.py:149-153)
      const float4* cr = reinterpret_cast<const float4*>(p.ctx1_in + ((long long)n * 2 + (t + 2)) * 512);
#pragma unroll
      for (int i = 0; i < 4; ++i) dst[i * 32 + lane] = cr[i * 32 + lane];
    } else {
#pragma unroll
      for (int i = 0; i < 4; ++i) dst[i * 32 + lane] = make_float4(0, 0, 0, 0);
    }
  }
  __syncthreads();

  // ---- phase 2: thread = channel c; both depthwise convs + GELU + group sum + skip.
  // The four channel multipliers are handled as two fp32 pairs (fma2_rn: IEEE FMAs, same results
  // as scalar fmaf), plus the 8 MUFU (ex2, rcp) per channel and frame.
  float2 w1p[2][3], w2p[2][3], b1p[2], b2p[2];  // [pair (m0,m1) / (m2,m3)][tap]
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    b1p[h] = make_float2(p.b1[4 * c + 2 * h], p.b1[4 * c + 2 * h + 1]);
    b2p[h] = make_float2(p.b2[4 * c + 2 * h], p.b2[4 * c + 2 * h + 1]);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      w1p[h][k] = make_float2(p.w1[(4 * c + 2 * h) * 3 + k], p.w1[(4 * c + 2 * h + 1) * 3 + k]);
      w2p[h][k] = make_float2(p.w2[(4 * c + 2 * h) * 3 + k], p.w2[(4 * c + 2 * h + 1) * 3 + k]);
    }
  }
  // h1 of frame f = first + j is a function of smem rows j, j+1, j+2 (both modes)
  const int first = CAUSAL ? t0 - 2 : t0 - 1;
  auto per_query = [&](const int q, const float4 (&ctx_cur)[2]) {
    const int n = n0 + q;
    float* yq = ybuf + q * RY * 512 + c;
    if (CAUSAL && p.ctx1_out != nullptr) {
      // new context of the layer-normed input: last two frames of [ctx | y] (nets.py:153);
      // written before the rows are recycled for z
      for (int t = max(t0, T - 2); t < t1; ++t)
        p.ctx1_out[((long long)n * 2 + (t - (T - 2))) * 512 + c] = yq[(t - lo) * 512];
      // clip shorter than the context: slot 0 <- old frame -1, which phase 1 staged in row 3
      // (frame -1) of this query; reading the staged copy (not ctx1_in) keeps the update correct
      // when the caller passes the SAME buffers as context in and out (streaming, T = 1)
      if (T == 1 && t0 == 0) p.ctx1_out[((long long)n * 2) * 512 + c] = yq[3 * 512];
    }
    float y0 = yq[0], y1 = yq[512];
    float2 ha[2], hb[2], hc[2];  // h1 of three consecutive frames, [pair]
    // h1 of frame f = first + j.  The tested form handles sequence ends (zero padding / causal
    // context / context output); the untested form is the same arithmetic without the tests, so a
    // frame gives the same bits whichever form computes it (chunk invariance stays exact).
    auto h1_math = [&](float y2, float2 (&o)[2]) {
      const float2 Y0 = make_float2(y0, y0), Y1 = make_float2(y1, y1), Y2 = make_float2(y2, y2);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const float2 a = fma2_rn(w1p[h][2], Y2, fma2_rn(w1p[h][1], Y1, fma2_rn(w1p[h][0], Y0, b1p[h])));
        o[h] = gelu_tanh2(a);
      }
    };
    auto h1 = [&](int j, float2 (&o)[2]) {
      const int f = first + j;
      const float y2 = yq[(j + 2) * 512];
      if (f >= 0 && f < T) {
        h1_math(y2, o);
        if (CAUSAL && p.ctx2_out != nullptr && f >= T - 2)  // last two frames of [ctx | h1] (nets.py:167)
          *reinterpret_cast<float4*>(p.ctx2_out + ((long long)n * 2 + (f - (T - 2))) * 2048 + 4 * c) =
              make_float4(o[0].x, o[0].y, o[1].x, o[1].y);
      } else if (has_ctx2 && f >= -2 && f < 0) {
        const float4 v = SMALL ? ((f == -2) ? ctx_cur[0] : ctx_cur[1])
                               : *reinterpret_cast<const float4*>(p.ctx2_in + ((long long)n * 2 + (f + 2)) * 2048 + 4 * c);
        o[0] = make_float2(v.x, v.y);
        o[1] = make_float2(v.z, v.w);
      } else {
        o[0] = o[1] = make_float2(0.f, 0.f);  // zero padding of the second conv's input
      }
      y0 = y1;
      y1 = y2;
    };
    // second conv + group sum + skip for output frame i, from h1 of frames i-1, i, i+1 (a, b, c);
    // rows <= i + 2 of this column are dead by then: z[t0 + i] is parked in row i.  Summation
    // order of the reference (nets.py:178-180): ((m0 + m1) + m2) + m3, then + skip.
    auto emit = [&](float* yrow, const float* xrow, float* zrow, const float2 (&a)[2],
                    const float2 (&b)[2], const float2 (&cc)[2]) {
      float2 t[2];
#pragma unroll
      for (int h = 0; h < 2; ++h)
        t[h] = fma2_rn(w2p[h][2], cc[h], fma2_rn(w2p[h][1], b[h], fma2_rn(w2p[h][0], a[h], b2p[h])));
      const float acc = (((t[0].x + t[0].y) + t[1].x) + t[1].y) + *xrow;
      *yrow = acc;
      *zrow = acc;
    };
    h1(0, ha);
    h1(1, hb);
    // T = 1: hb is h1 of frame -1 (old context slot 1, or zero); it becomes slot 0 of the new
    // context.  Written only now, after both old slots were read (in/out buffers may alias).
    if (CAUSAL && p.ctx2_out != nullptr && T == 1 && t0 == 0)
      *reinterpret_cast<float4*>(p.ctx2_out + ((long long)n * 2) * 2048 + 4 * c) =
          make_float4(hb[0].x, hb[0].y, hb[1].x, hb[1].y);
    const int nout = t1 - t0;
    // output frames whose newest h1 frame (first + i + 2) needs no end-of-sequence handling
    int i_lo = max(0, -(first + 2));
    int i_hi = min(nout, ((CAUSAL && p.ctx2_out != nullptr) ? T - 2 : T) - (first + 2));
    if (i_hi < i_lo) i_lo = i_hi = 0;
    float* yp = yq;
    const float* xp = xraw + q * TT * 512 + c;
    float* zp = p.z + ((long long)n * T + t0) * 512 + c;
    int i = 0;
    auto checked_until = [&](int stop) {
      for (; i < stop; ++i, yp += 512, xp += 512, zp += 512) {
        h1(i + 2, hc);
        emit(yp, xp, zp, ha, hb, hc);
#pragma unroll
        for (int h = 0; h < 2; ++h) { ha[h] = hb[h]; hb[h] = hc[h]; }
      }
    };
    checked_until(i_lo);
    // interior, three frames per trip: the roles of (ha, hb, hc) rotate back after three steps,
    // so no register moves and no tests
    for (; i + 3 <= i_hi; i += 3, yp += 1536, xp += 1536, zp += 1536) {
      const float ya = yp[4 * 512], yb = yp[5 * 512], yc = yp[6 * 512];
      h1_math(ya, hc);
      y0 = y1; y1 = ya;
      emit(yp, xp, zp, ha, hb, hc);
      h1_math(yb, ha);
      y0 = y1; y1 = yb;
      emit(yp + 512, xp + 512, zp + 512, hb, hc, ha);
      h1_math(yc, hb);
      y0 = y1; y1 = yc;
      emit(yp + 1024, xp + 1024, zp + 1024, hc, ha, hb);
    }
    checked_until(nout);
  };
  if constexpr (SMALL) {
    // unrolled so that each copy indexes ctx_all with a constant (it must stay in registers)
#pragma unroll
    for (int q = 0; q < kDwSmallQueries; ++q) {
      if (q < nq) {
        const float4 cur[2] = {ctx_all[q % kDwCtxWindow][0], ctx_all[q % kDwCtxWindow][1]};
        if (q + kDwCtxWindow < kDwSmallQueries) fetch_ctx2(q + kDwCtxWindow, ctx_all[q % kDwCtxWindow]);
        per_query(q, cur);
      }
    }
  } else {
    for (int q = 0; q < nq; ++q) per_query(q, ctx_all[0]);
  }
  __syncthreads();

  // ---- phase 3: LN_1(z) * w (scale only) -> bf16 planes, the A operand of the `up` GEMM
  const int ntile = t1 - t0;
  for (int rq = warp; rq < nq * ntile; rq += 16) {
    const int q = rq / ntile, i = rq - q * ntile;
    const float4* zr = reinterpret_cast<const float4*>(ybuf + (q * RY + i) * 512);
    float4 v[4], o4[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) v[k] = zr[k * 32 + lane];
    ln512(v, p.ln1_w, lane, o4);
    const long long orow = (long long)(n0 + q) * T + t0 + i;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      float o[4] = {o4[k].x, o4[k].y, o4[k].z, o4[k].w};
      for (int pl = 0; pl < p.planes; ++pl) {
        uint2 pk;
        pk.x = bf16x2_split(o[0], o[1]);
        pk.y = bf16x2_split(o[2], o[3]);
        *reinterpret_cast<uint2*>(p.planes_out + pl * p.plane_stride + orow * 512 + (k * 32 + lane) * 4) = pk;
      }
    }
  }
}

// ------------------------------------------------------------------------ a7 epilogue
// video_hw (nullable): per-clip video sizes [clips][2], clip = row / rows_per_clip, or
// query_clip[query] when query_clip is not null
__global__ void __launch_bounds__(128) refine_update_kernel(const tapir_update_args a,
                                                            const int32_t* __restrict__ video_hw,
                                                            long long rows_per_clip,
                                                            const int32_t* __restrict__ query_clip) {
  const long long row = blockIdx.x;
  const int T = a.num_frames;
  const int n = (int)(row / T), t = (int)(row - (long long)n * T);
  const float* res = a.res + row * a.ld_res;
  const float* fhi = a.feat_hi + n * a.feat_hi_stride_n + t * a.feat_hi_stride_t;
  const float* flo = a.feat_lo + n * a.feat_lo_stride_n + t * a.feat_lo_stride_t;
  for (int e = threadIdx.x; e < 384; e += blockDim.x) {
    const float f = (e < 128) ? fhi[e] : flo[e - 128];
    a.feat_out[row * 384 + e] = res[4 + e] + f;
  }
  if (threadIdx.x == 0) {
    // tapir_model.py:674-682: delta is in resized-resolution pixels -> initial_resolution
    const float dx = __fdiv_rn(__fmul_rn(res[0], (float)a.init_w), (float)a.resize_w);
    const float dy = __fdiv_rn(__fmul_rn(res[1], (float)a.init_h), (float)a.resize_h);
    const float x = dx + a.pos[row * 2 + 0], y = dy + a.pos[row * 2 + 1];
    a.pos[row * 2 + 0] = x;
    a.pos[row * 2 + 1] = y;
    a.occ_out[row] = res[2] + a.occ_in[row];
    a.expd_out[row] = res[3] + a.expd_in[row];
    if (a.tracks_out != nullptr) {
      int vh = a.video_h, vw = a.video_w;
      if (video_hw != nullptr) {
        const long long clip = query_clip != nullptr ? query_clip[n] : row / rows_per_clip;
        vh = video_hw[clip * 2 + 0];
        vw = video_hw[clip * 2 + 1];
      }
      // train2orig (tapir_model.py:435-441)
      a.tracks_out[row * 2 + 0] = __fdiv_rn(__fmul_rn(x, (float)vw), (float)a.init_w);
      a.tracks_out[row * 2 + 1] = __fdiv_rn(__fmul_rn(y, (float)vh), (float)a.init_h);
    }
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

int pool_pyramid(const float* grid, int T, int h, int w, int C, float* out, cudaStream_t s) {
  TAPIR_CHECK_ARG(grid && out && T > 0 && h >= 2 && w >= 2 && C % 4 == 0, "pool_pyramid: bad arguments");
  const long long total = (long long)T * (h / 2) * (w / 2) * (C / 4);
  ProfileScope ps("pool_pyramid", s, 0.0, (double)total * 16 * 5);
  pool_kernel<<<grid_for(total), 256, 0, s>>>(reinterpret_cast<const float4*>(grid), h, w, C / 4,
                                             reinterpret_cast<float4*>(out), total);
  count_launch();
  TAPIR_LAUNCH_CHECK("pool_kernel");
  return kOk;
}

int local_corr(const tapir_corr_args* a, int batch, cudaStream_t s, const int32_t* query_clip) {
  TAPIR_CHECK_ARG(a != nullptr && a->num_levels >= 1 && a->num_levels <= TAPIR_MAX_CORR_LEVELS,
                  "local_corr: bad level count");
  TAPIR_CHECK_ARG(batch >= 1, "local_corr: bad clip count %d", batch);
  TAPIR_CHECK_ARG(a->pos && a->occ && a->expd && a->feat_hi && a->feat_lo && a->out_planes,
                  "local_corr: null pointer");
  TAPIR_CHECK_ARG(a->planes >= 1 && a->planes <= 3 && a->num_points > 0 && a->num_frames > 0,
                  "local_corr: bad shape");
  TAPIR_CHECK_ARG(a->ld >= 388 + 49 * a->num_levels && a->ld % 8 == 0, "local_corr: ld=%d too small", a->ld);
  for (int l = 0; l < a->num_levels; ++l) {
    const tapir_corr_level& L = a->levels[l];
    TAPIR_CHECK_ARG(L.grid != nullptr && (L.C == 128 || L.C == 256), "local_corr: level %d C=%d unsupported", l, L.C);
    TAPIR_CHECK_ARG((l == 0) == (L.C == 128), "local_corr: level 0 must be the 128-ch hires grid, others 256-ch");
    // (x spacing of the 49 samples is gw/gh cells - a reference quirk; boxes wider than the
    // 16-column table take the per-sample path inside the kernel)
  }
  const long long rows = (long long)a->num_points * (query_clip != nullptr ? 1 : batch) * a->num_frames;
  TAPIR_CHECK_ARG(rows < (1ll << 31), "local_corr: %lld rows exceed one launch", rows);
  CorrParams p;
  p.a = *a;
  p.batch = batch;
  p.query_clip = query_clip;
  double cell_bytes = 0;
  for (int l = 0; l < a->num_levels; ++l) cell_bytes += 64.0 * a->levels[l].C * 4;
  // SURVEY.md 8(d): N*T*(64 cells * sum C * e + 384*4 + 8 + 147*4)
  ProfileScope ps("local_corr", s, (double)rows * (cell_bytes / 2 + 1200),
                  (double)rows * (cell_bytes + 384 * 4 + 8 + 49.0 * a->num_levels * 4));
  local_corr_kernel<<<(unsigned)rows, 32 * a->num_levels, 0, s>>>(p);  // one warp per pyramid level
  count_launch();
  TAPIR_LAUNCH_CHECK("local_corr_kernel");
  return kOk;
}

int refine_update(const tapir_update_args* a, cudaStream_t s, const int32_t* video_hw,
                  long long rows_per_clip, const int32_t* query_clip) {
  TAPIR_CHECK_ARG(a != nullptr && a->res && a->pos && a->feat_out && a->occ_out && a->expd_out,
                  "refine_update: null pointer");
  const long long rows = (long long)a->num_points * a->num_frames;
  ProfileScope ps("refine_update", s, 0.0, (double)rows * (388 * 4 + 384 * 8));
  refine_update_kernel<<<(unsigned)rows, 128, 0, s>>>(*a, video_hw, rows_per_clip, query_clip);
  count_launch();
  TAPIR_LAUNCH_CHECK("refine_update_kernel");
  return kOk;
}

// ------------------------------------------------------------------------ mixer orchestration

namespace {
struct MixerPlan {
  float* xa;   // residual stream [rows][512]
  float* xb;
  __nv_bfloat16* y;  // [P][rows][512]
  __nv_bfloat16* h;  // [P][rows][2048]
  float* splitk;     // split-K scratch (streaming / tiny batches)
};
constexpr size_t kSplitKBytes = 40u << 20;
size_t plan_mixer(Arena& a, long long rows, int planes, MixerPlan* m) {
  m->xa = a.take<float>((size_t)rows * 512);
  m->xb = a.take<float>((size_t)rows * 512);
  m->y = a.take<__nv_bfloat16>((size_t)rows * 512 * planes);
  m->h = a.take<__nv_bfloat16>((size_t)rows * 2048 * planes);
  m->splitk = a.take<float>(kSplitKBytes / sizeof(float));
  return a.off;
}
// A mixer GEMM: split-K only for single-frame (streaming) steps, see GemmArgs::allow_splitk.
GemmArgs mixer_gemm_args(const tapir_linear& l, const MixerPlan& m, int T) {
  GemmArgs g = gemm_args(l);
  g.splitk_ws = m.splitk; g.splitk_ws_bytes = kSplitKBytes; g.allow_splitk = (T == 1);
  return g;
}
}  // namespace

int mixer_dw(const tapir_mixer_block& blk, const float* x, int n, int T, bool causal, const float* ctx1_in,
             const float* ctx2_in, float* ctx1_out, float* ctx2_out, float* z, __nv_bfloat16* planes_out,
             long long plane_stride, int planes, cudaStream_t s) {
  static PerDeviceOnce configured;
  if (configured.pending()) {
    const int max_smem = kDwRowBudget * 512 * (int)sizeof(float);
    TAPIR_CUDA(cudaFuncSetAttribute(mixer_dw_kernel<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem));
    TAPIR_CUDA(cudaFuncSetAttribute(mixer_dw_kernel<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem));
    TAPIR_CUDA(cudaFuncSetAttribute(mixer_dw_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem));
    configured.mark();
  }
  const long long rows = (long long)n * T;
  DwParams d;
  d.x = x; d.z = z;
  d.planes_out = planes_out; d.plane_stride = plane_stride; d.planes = planes;
  d.T = T; d.N = n;
  d.TT = T < kDwTileMax ? T : kDwTileMax;
  d.QB = kDwRowBudget / (2 * d.TT + kDwHalo);
  if (d.QB < 1) d.QB = 1;
  if (d.QB > kDwSmallQueries) d.QB = kDwSmallQueries;
  // few rows in total (streaming): fewer queries per CTA so that every SM gets one
  // (the several-queries-per-CTA variant runs one CTA per SM: aim at exactly one round)
  if (d.QB > 1) {
    const long long per_sm = ceil_div_ll((long long)n * ceil_div(T, d.TT), num_sms());
    if (per_sm < d.QB) d.QB = per_sm < 2 ? 2 : (int)per_sm;
  }
  if (d.QB > n) d.QB = n;
  d.ln_w = blk.ln_w; d.w1 = blk.dw1_w; d.b1 = blk.dw1_b; d.w2 = blk.dw2_w; d.b2 = blk.dw2_b;
  d.ln1_w = blk.ln1_w;
  d.ctx1_in = ctx1_in;
  d.ctx2_in = ctx2_in;
  d.ctx1_out = ctx1_out;
  d.ctx2_out = ctx2_out;
  dim3 grid(ceil_div(T, d.TT), ceil_div(n, d.QB));
  const int dw_smem = d.QB * (2 * d.TT + kDwHalo) * 512 * (int)sizeof(float);
  {
    ProfileScope ps("mixer.dw", s, (double)rows * 2048 * 12, (double)rows * 512 * (8 + 2 * planes));
    // SMALL exists for the causal context prefetch.  Its non-causal instantiation is miscompiled
    // for sm_90 by CUDA 12.9 ptxas (-O1 and up, query loop unrolled): wrong outputs for tiles of
    // 5+ frames, right at -O0 or not unrolled.  Non-causal tiles run the generic kernel; the
    // causal one is checked over the same code paths (test_mixer_causal_with_context).
    if (causal) {
      if (d.QB > 1) mixer_dw_kernel<true, true><<<grid, 512, dw_smem, s>>>(d);
      else mixer_dw_kernel<true, false><<<grid, 512, dw_smem, s>>>(d);
    } else {
      mixer_dw_kernel<false, false><<<grid, 512, dw_smem, s>>>(d);
    }
  }
  count_launch();
  TAPIR_LAUNCH_CHECK("mixer_dw_kernel");
  return kOk;
}

size_t mixer_workspace_bytes(long long rows, int planes) {
  Arena a(nullptr, 0);
  MixerPlan m;
  return plan_mixer(a, rows, planes, &m) + 256;
}

int mixer_forward(const tapir_mixer_weights* w, const tapir_mixer_io* io, void* ws, size_t ws_bytes,
                  cudaStream_t s) {
  TAPIR_CHECK_ARG(w && io && io->x_planes && io->out, "mixer_forward: null pointer");
  const int P = w->planes;
  const int n = io->num_points, T = io->num_frames;
  const long long rows = (long long)n * T;
  TAPIR_CHECK_ARG(n > 0 && T > 0 && n <= 65535, "mixer_forward: bad shape n=%d T=%d", n, T);
  TAPIR_CHECK_ARG(w->num_blocks >= 1 && w->num_blocks <= TAPIR_MAX_MIXER_BLOCKS, "mixer_forward: num_blocks");
  TAPIR_CHECK_ARG(io->ldx == w->linear.K, "mixer_forward: ldx=%d must equal the padded input width %d", io->ldx, w->linear.K);
  TAPIR_CHECK_ARG(io->ldo >= w->linear_1.N, "mixer_forward: ldo too small");
  Arena arena(ws, ws_bytes);
  MixerPlan m;
  plan_mixer(arena, rows, P, &m);
  if (!arena.ok) {
    set_error("mixer_forward: workspace too small (%zu < %zu)", ws_bytes, arena.off);
    return kWorkspaceTooSmall;
  }
  {  // nets.py:235 linear
    GemmArgs g = mixer_gemm_args(w->linear, m, T);
    g.tag = "mixer.linear_in";
    g.M = (int)rows;
    g.a = static_cast<const __nv_bfloat16*>(io->x_planes);
    g.lda = io->ldx;
    g.a_plane_stride = io->x_plane_stride;
    g.out_f32 = m.xa; g.ldo = 512;
    TAPIR_RETURN_IF(gemm(g, s));
  }
  for (int b = 0; b < w->num_blocks; ++b) {
    const tapir_mixer_block& blk = w->blocks[b];
    TAPIR_RETURN_IF(mixer_dw(blk, m.xa, n, T, io->causal != 0, io->ctx1_in ? io->ctx1_in[b] : nullptr,
                             io->ctx2_in ? io->ctx2_in[b] : nullptr, io->ctx1_out ? io->ctx1_out[b] : nullptr,
                             io->ctx2_out ? io->ctx2_out[b] : nullptr, m.xb, m.y, rows * 512, P, s));
    {
      GemmArgs g = mixer_gemm_args(blk.up, m, T);
      g.tag = "mixer.up";
      g.M = (int)rows;
      g.a = m.y; g.lda = 512; g.a_plane_stride = rows * 512;
      g.act = 1;
      g.out_planes = m.h; g.ldp = 2048; g.out_plane_stride = rows * 2048; g.out_P = P;
      TAPIR_RETURN_IF(gemm(g, s));
    }
    {
      GemmArgs g = mixer_gemm_args(blk.down, m, T);
      g.tag = "mixer.down";
      g.M = (int)rows;
      g.a = m.h; g.lda = 2048; g.a_plane_stride = rows * 2048;
      g.residual = m.xb; g.ldr = 512;
      g.out_f32 = m.xa; g.ldo = 512;
      TAPIR_RETURN_IF(gemm(g, s));
    }
  }
  TAPIR_RETURN_IF(layernorm_split(m.xa, rows, 512, w->ln_w, nullptr, nullptr, m.y, rows * 512, P, s));
  {
    GemmArgs g = mixer_gemm_args(w->linear_1, m, T);
    g.tag = "mixer.linear_out";
    g.M = (int)rows;
    g.a = m.y; g.lda = 512; g.a_plane_stride = rows * 512;
    g.out_f32 = io->out; g.ldo = io->ldo;
    TAPIR_RETURN_IF(gemm(g, s));
  }
  return kOk;
}

}  // namespace tapir
