// Stage A (SURVEY.md 8(a4),(a6)): query-feature sampling, global cost volume and the
// track / occlusion head.
//
// The cost volume itself is the split-bf16 wgmma GEMM (planes=3, i.e. fp32-equivalent,
// because its arg-max must match the reference bit-exactly): cv[n][t*h*w + cell] with
// M = queries, N = T*h*w cells, K = 256.  A head kernel then turns every map into a track point:
// conv3x3 1->16 + ReLU, conv3x3 16->1, temperature soft-max, arg-max, radius-5 soft arg-max, and
// the occlusion branch (pad(0,2,0,2), conv3x3 stride 2 16->32 + ReLU, spatial mean, 32->16->2
// MLP).  32x32 maps (initial_resolution 256 x 256) run `cost_volume_head_tc_kernel`, one map at a
// time per persistent CTA from shared memory with the strided conv on the tensor cores; every
// other map size runs `cost_volume_head_generic_kernel`.
#include <cfloat>

#include "kernels.cuh"

namespace tapir {

namespace {

// ------------------------------------------------------------------------ a4
// utils.py:45-73 map_coordinates_3d: grid_sample(5-D, bilinear, align_corners=False,
// padding_mode='border') at (t+0.5, y, x) / (T, h, w).  We mirror ATen's arithmetic:
// g = 2*(c/size) - 1 ; pix = ((g + 1) * size - 1) / 2 ; clamp to [0, size-1].
__device__ __forceinline__ float unnormalize_border(float c, int size) {
  const float fs = (float)size;
  const float g = __fsub_rn(__fmul_rn(2.f, __fdiv_rn(c, fs)), 1.f);
  float pix = __fdiv_rn(__fsub_rn(__fmul_rn(__fadd_rn(g, 1.f), fs), 1.f), 2.f);
  pix = fminf(fmaxf(pix, 0.f), fs - 1.f);
  return pix;
}

// One query's features: the block's threads sample `grid` at (qt, qy, qx) into out[0 .. C).
// Ta: the clip length the coordinates are normalised by.  frame_slot: null for a grid holding all
// Ta frames (T == Ta), else Ta entries mapping each frame to its slot among the grid's T, or -1.  A
// tap of nonzero weight on a frame without a slot makes the query's row NaN: the grid is never read
// outside its T slots and a partial sum is never returned.
__device__ __forceinline__ void sample_query_row(const float* __restrict__ grid, int T, int gh, int gw,
                                                 int C, float qt, float qy, float qx, int vT, int vH,
                                                 int vW, int Ta, const int* __restrict__ frame_slot,
                                                 float* __restrict__ out) {
  // utils.convert_grid_coordinates: coords * out / in (tapir_model.py:266-277)
  float t = __fdiv_rn(__fmul_rn(qt, (float)Ta), (float)vT);
  const float y = __fdiv_rn(__fmul_rn(qy, (float)gh), (float)vH);
  const float x = __fdiv_rn(__fmul_rn(qx, (float)gw), (float)vW);
  t = __fadd_rn(t, 0.5f);
  const float pt = unnormalize_border(t, Ta), py = unnormalize_border(y, gh), px = unnormalize_border(x, gw);
  const int t0 = (int)floorf(pt), y0 = (int)floorf(py), x0 = (int)floorf(px);
  const float ft = pt - t0, fy = py - y0, fx = px - x0;
  bool in_clip[2];
  int slot[2];
#pragma unroll
  for (int dt = 0; dt < 2; ++dt) {
    const int tt = t0 + dt;
    in_clip[dt] = tt >= 0 && tt < Ta;
    slot[dt] = !in_clip[dt] ? -1 : frame_slot ? frame_slot[tt] : tt;
  }
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float acc = 0.f;
    bool missing = false;
#pragma unroll
    for (int dt = 0; dt < 2; ++dt)
#pragma unroll
      for (int dy = 0; dy < 2; ++dy)
#pragma unroll
        for (int dx = 0; dx < 2; ++dx) {
          const int tt = slot[dt], yy = y0 + dy, xx = x0 + dx;
          const float wgt = (dt ? ft : 1.f - ft) * (dy ? fy : 1.f - fy) * (dx ? fx : 1.f - fx);
          if (!in_clip[dt] || yy >= gh || xx >= gw || yy < 0 || xx < 0) continue;
          if (tt >= 0 && tt < T)
            acc += wgt * grid[(((long long)tt * gh + yy) * gw + xx) * C + c];
          else if (wgt != 0.f)
            missing = true;
        }
    out[c] = missing ? __int_as_float(0x7fc00000) : acc;
  }
}

__global__ void __launch_bounds__(128) sample_query_kernel(const float* __restrict__ grid, int T,
                                                           int gh, int gw, int C,
                                                           const float* __restrict__ q, int vT,
                                                           int vH, int vW, int Ta,
                                                           const int* __restrict__ frame_slot,
                                                           float* __restrict__ out) {
  const int n = blockIdx.x;
  sample_query_row(grid, T, gh, gw, C, q[n * 3 + 0], q[n * 3 + 1], q[n * 3 + 2], vT, vH, vW, Ta,
                   frame_slot, out + (long long)n * C);
}

// Point edits of a one-frame step (OnlineTracker.retarget / add_points): request r < *count
// re-samples row req[r].row of every query-feature grid from clip req[r].clip's grids, as
// sample_query_kernel does for a one-frame clip (T = vT = Ta = 1), and zeroes that row of every
// causal-state tensor.  blockIdx.y == 0 samples, blockIdx.y == 1 + k zeroes state tensor k (even
// k: [rows][2][512], odd k: [rows][2][2048]).  CTAs stride over the requests; with no request every
// CTA exits after one load.
struct QueryRowsParams {
  tapir_query_grid grids[TAPIR_MAX_QUERY_GRIDS];
  int num_grids, clips, rows, video_h, video_w;
  const int32_t* video_hw;  // [clips][2] or null (video_h x video_w for every clip)
  const int32_t* count;
  const tapir_query_request* req;
  float* const* state;
};

__global__ void __launch_bounds__(128) sample_query_rows_kernel(const QueryRowsParams p) {
  const int count = min(*p.count, p.rows);
  for (int r = blockIdx.x; r < count; r += gridDim.x) {
    const tapir_query_request q = p.req[r];
    if (q.row < 0 || q.row >= p.rows || q.clip < 0 || q.clip >= p.clips) continue;
    if (blockIdx.y == 0) {
      const int vh = p.video_hw ? p.video_hw[q.clip * 2 + 0] : p.video_h;
      const int vw = p.video_hw ? p.video_hw[q.clip * 2 + 1] : p.video_w;
      // constant indices: the grid table stays in the parameter space
#pragma unroll
      for (int i = 0; i < TAPIR_MAX_QUERY_GRIDS; ++i) {
        if (i >= p.num_grids) break;
        const tapir_query_grid g = p.grids[i];
        sample_query_row(g.grid + q.clip * g.clip_stride, 1, g.h, g.w, g.C, q.t, q.y, q.x, 1, vh, vw, 1,
                         nullptr, g.out + (long long)q.row * g.C);
      }
    } else {
      const int k = blockIdx.y - 1;
      const int width4 = (k & 1) ? 2 * 2048 / 4 : 2 * 512 / 4;
      float4* dst = reinterpret_cast<float4*>(p.state[k]) + (long long)q.row * width4;
      for (int i = threadIdx.x; i < width4; i += blockDim.x) dst[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
}

// ------------------------------------------------------------------------ a6 head, shared parts
// Single-barrier block reductions over NW warps: each warp's result goes to the reduction's own
// slot, then EVERY thread folds the NW partials itself in ascending warp order (broadcast loads
// instead of two more barriers; the tensor-core head spent 21 % of its stall samples on
// barriers).  A head gives each reduction of a map its own slot and writes a slot again only in
// the next map, after at least one more __syncthreads, so that write comes after every read.
template <int NW>
struct RedSlot {
  float f[NW * 3];
  int i[NW];
};

// maximum value; among equal values the LOWEST index (torch.argmax on CPU)
template <int NW>
__device__ __forceinline__ void block_max_first(float v, int idx, RedSlot<NW>& s, float* out_v,
                                                int* out_i) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, v, o);
    const int oi = __shfl_xor_sync(0xffffffffu, idx, o);
    if (ov > v || (ov == v && oi < idx)) { v = ov; idx = oi; }
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) { s.f[warp] = v; s.i[warp] = idx; }
  __syncthreads();
  float bv = s.f[0];
  int bi = s.i[0];
#pragma unroll
  for (int k = 1; k < NW; ++k) {
    const float kv = s.f[k];
    const int ki = s.i[k];
    if (kv > bv || (kv == bv && ki < bi)) { bv = kv; bi = ki; }
  }
  *out_v = bv;
  *out_i = bi;
}

template <int NW>
__device__ __forceinline__ void block_sum3(float a, float b, float c, RedSlot<NW>& s, float* oa,
                                           float* ob, float* oc) {
  a = warp_sum(a); b = warp_sum(b); c = warp_sum(c);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) { s.f[warp * 3] = a; s.f[warp * 3 + 1] = b; s.f[warp * 3 + 2] = c; }
  __syncthreads();
  float x = 0, y = 0, z = 0;
#pragma unroll
  for (int k = 0; k < NW; ++k) { x += s.f[k * 3]; y += s.f[k * 3 + 1]; z += s.f[k * 3 + 2]; }
  *oa = x; *ob = y; *oc = z;
}

// The rest of map (n, t) after the spatial mean of hid3, run by warp 0 alone with shuffles
// (lane = channel of `mean`): hid4 32 -> 16 + ReLU, occ_out 16 -> 2, the soft arg-max (tx, ty) / tw
// of a gh x gw map scaled to initial_resolution pixels, the query-frame passthrough and the
// stores.  w4, b4, w5, b5 are the hid4 and occ_out weights.
__device__ __forceinline__ void head_tail(float mean, const float* w4, const float* b4, const float* w5,
                                          const float* b5, float tx, float ty, float tw, int am, int gh,
                                          int gw, int n, int t, int T, const float* query_tyx, int init_h,
                                          int init_w, float* points, float* occ_out, float* expd_out,
                                          int* argmax_out) {
  const int lane = threadIdx.x & 31;
  float a = (lane < 16) ? b4[lane] : 0.f;  // hid4: 32 -> 16, ReLU
#pragma unroll
  for (int k = 0; k < 32; ++k) {
    const float mk = __shfl_sync(0xffffffffu, mean, k);
    if (lane < 16) a = fmaf(mk, w4[lane * 32 + k], a);
  }
  a = fmaxf(a, 0.f);
  float o2 = (lane < 2) ? b5[lane] : 0.f;  // occ_out: 16 -> 2
#pragma unroll
  for (int k = 0; k < 16; ++k) {
    const float hk = __shfl_sync(0xffffffffu, a, k);
    if (lane < 2) o2 = fmaf(hk, w5[lane * 16 + k], o2);
  }
  const long long o = (long long)n * T + t;
  if (lane == 0) occ_out[o] = o2;
  if (lane == 1) expd_out[o] = o2;
  if (lane == 0) {
    const float den = fmaxf(tw, 1e-12f);
    // utils.py:165-169: cell units -> initial_resolution pixels (coords * out / in)
    float px = __fdiv_rn(__fmul_rn(tx / den, (float)init_w), (float)gw);
    float py = __fdiv_rn(__fmul_rn(ty / den, (float)init_h), (float)gh);
    if (query_tyx != nullptr) {
      // utils.py:171-191: on the query frame the track passes through the query point
      const float qf = rintf(query_tyx[n * 3 + 0]);
      if (qf == (float)t) { px = query_tyx[n * 3 + 2]; py = query_tyx[n * 3 + 1]; }
    }
    points[o * 2 + 0] = px;
    points[o * 2 + 1] = py;
    if (argmax_out != nullptr) argmax_out[o] = am;
  }
}

// ------------------------------------------------------------------------ a6 head, 32 x 32 maps
// One persistent CTA per SM walks the maps.  The 16->32 stride-2 conv (80 % of the head FLOPs)
// runs on the tensor cores as a split-bf16 implicit GEMM per map:
// M = 256 output pixels, N = 32 channels, K = 9 taps x 16 input channels (one m16n8k16 k-step per
// tap), three MMAs per product (hi*hi + hi*lo + lo*hi), fp32 accumulation.  ReLU(hid1) is kept as
// bf16 hi/lo planes in channel-last order (A fragments are plain 32-bit shared loads), and the
// 16->1 conv is evaluated in exact fp32 from registers as nine per-tap channel dot products
// (`stap`) that are then gathered - so the soft-argmax path never sees bf16.
constexpr int kG = 32;            // cost-volume map side (initial_resolution 256 / stride 8)
constexpr int kOccW = kG + 3;     // 35: index -1 .. 33 (1 left halo for hid2, 2 right for hid3)
constexpr int kOccPlane = kOccW * kOccW;
constexpr int kHT = 512;                       // threads per map
constexpr int kPixW = 9;                       // 32-bit words per pixel: 16 bf16 + 1 pad (bank spread)
constexpr int kPlaneWords = kOccPlane * kPixW; // 35 x 35 pixels
constexpr int kTapW = (kG + 2) * (kG + 2);

// kW3Stride = 32-bit words per hid3 weight row.  With the pixel stride (9) every weight-fragment
// load of phase D was 2-way bank conflicted (lane group g = 7 lands on the banks of g = 0: 49 M of
// the 145 M shared wavefronts per launch); 12 makes {12 g + tq} distinct mod 32.
constexpr int kW3Stride = 12;
struct HeadTcSmem {
  float cv[kTapW];
  float stap[9 * kTapW];
  uint32_t occ_hi[kPlaneWords], occ_lo[kPlaneWords];
  uint32_t w3_hi[9 * 32 * kW3Stride], w3_lo[9 * 32 * kW3Stride];  // [tap][co][ci pairs]
  // hid1 / hid2 weights, 9 taps padded to 12 per channel: three broadcast LDS.128 per channel
  __align__(16) float w1[16 * 12];
  __align__(16) float w2[16 * 12];
  float b1[16], b3[32];
  float w4[16 * 32], b4[16], w5[2 * 16], b5[2];
  float mean32[16][32];
  // one slot per block reduction of a map (4 per map): a slot is rewritten only in the next map,
  // after the barrier before the tail and the barrier that publishes the next map
  RedSlot<16> slot[4];
};

__device__ __forceinline__ void mma_bf16_16816(float (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
      "{%0, %1, %2, %3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

static_assert(sizeof(HeadTcSmem) <= 227 * 1024, "head kernel shared memory exceeds the 227 KB opt-in limit");

__global__ void __launch_bounds__(kHT, 1) cost_volume_head_tc_kernel(
    const tapir_head_weights w, const float* __restrict__ cost_volume, int T, int num_maps,
    const float* __restrict__ query_tyx, float temperature, int init_h, int init_w,
    float* __restrict__ points, float* __restrict__ occ_out, float* __restrict__ expd_out,
    int* __restrict__ argmax_out) {
  extern __shared__ __align__(16) uint8_t head_tc_smem_raw[];
  HeadTcSmem& sm = *reinterpret_cast<HeadTcSmem*>(head_tc_smem_raw);
  const int tid = threadIdx.x;
  const int warp = tid >> 5, lane = tid & 31;

  // ---- phase A (once per persistent CTA): zero halos, stage weights (hid3 weights as bf16
  // hi/lo planes [tap][co][ci]); the interiors are fully rewritten for every map
  for (int i = tid; i < kTapW; i += kHT) sm.cv[i] = 0.f;
  for (int i = tid; i < 9 * kTapW; i += kHT) sm.stap[i] = 0.f;
  for (int i = tid; i < kPlaneWords; i += kHT) { sm.occ_hi[i] = 0u; sm.occ_lo[i] = 0u; }
  for (int i = tid; i < 9 * 32 * 8; i += kHT) {
    const int cp = i & 7, co = (i >> 3) & 31, tap = i >> 8;
    float v0 = w.hid3_w[(co * 16 + 2 * cp) * 9 + tap], v1 = w.hid3_w[(co * 16 + 2 * cp + 1) * 9 + tap];
    const uint32_t hi = bf16x2_split(v0, v1);
    const uint32_t lo = bf16x2_split(v0, v1);
    sm.w3_hi[(tap * 32 + co) * kW3Stride + cp] = hi;
    sm.w3_lo[(tap * 32 + co) * kW3Stride + cp] = lo;
  }
  if (tid < 192) {
    const int co = tid / 12, k = tid - co * 12;
    sm.w1[tid] = (k < 9) ? w.hid1_w[co * 9 + k] : 0.f;
    sm.w2[tid] = (k < 9) ? w.hid2_w[co * 9 + k] : 0.f;
  }
  if (tid < 16) { sm.b1[tid] = w.hid1_b[tid]; sm.b4[tid] = w.hid4_b[tid]; }
  if (tid < 32) { sm.b3[tid] = w.hid3_b[tid]; sm.w5[tid] = w.occ_w[tid]; }
  if (tid < 2) sm.b5[tid] = w.occ_b[tid];
  sm.w4[tid] = w.hid4_w[tid];

  // the next map's 4 KB are fetched into registers (2 floats per thread) while the current map
  // is processed, so the L2/HBM latency is not exposed between maps
  float2 pre = make_float2(0.f, 0.f);
  if ((int)blockIdx.x < num_maps)
    pre = reinterpret_cast<const float2*>(cost_volume + (long long)blockIdx.x * (kG * kG))[tid];
  __syncthreads();  // phase A's zero fill of `cv` is ordered before the first map's interior writes
  for (int map = blockIdx.x; map < num_maps; map += gridDim.x) {
  const int n = map / T, t = map - n * T;
  // (no barrier here: `cv` was last read in the previous map's phase B, several barriers ago;
  // the barrier below publishes the new map and, on the first trip, the staged weights)
  {
    const int i = 2 * tid;  // pixels i, i+1 of the 32x32 map (same row)
    float* d = sm.cv + ((i >> 5) + 1) * (kG + 2) + (i & 31) + 1;
    d[0] = pre.x;
    d[1] = pre.y;
    const int nxt = map + gridDim.x;
    if (nxt < num_maps) pre = reinterpret_cast<const float2*>(cost_volume + (long long)nxt * (kG * kG))[tid];
  }
  __syncthreads();

  // ---- phase B: hid1 (conv3x3 1->16, padding 1, ReLU) for 2 adjacent pixels of one row; the
  // 16 channel values go to the bf16 planes and into the nine per-tap dot products of hid2
  const int y = tid >> 4, x0 = (tid & 15) * 2;
  {
    float win[3][4];
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
      for (int c = 0; c < 4; ++c) win[r][c] = sm.cv[(y + r) * (kG + 2) + x0 + c];
    float st[2][9];
#pragma unroll
    for (int p = 0; p < 2; ++p)
#pragma unroll
      for (int k = 0; k < 9; ++k) st[p][k] = 0.f;
    const int pix0 = (y + 1) * kOccW + (x0 + 1);
#pragma unroll 2
    for (int cp = 0; cp < 8; ++cp) {
      float o[2][2];  // [pixel][channel of the pair]
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int co = 2 * cp + e;
        float a0 = sm.b1[co], a1 = a0;
        float wk[12];
#pragma unroll
        for (int v = 0; v < 3; ++v)
          *reinterpret_cast<float4*>(wk + 4 * v) = reinterpret_cast<const float4*>(sm.w1 + co * 12)[v];
#pragma unroll
        for (int ky = 0; ky < 3; ++ky)
#pragma unroll
          for (int kx = 0; kx < 3; ++kx) {
            const float wv = wk[ky * 3 + kx];
            a0 = fmaf(win[ky][kx], wv, a0);
            a1 = fmaf(win[ky][kx + 1], wv, a1);
          }
        o[0][e] = fmaxf(a0, 0.f);
        o[1][e] = fmaxf(a1, 0.f);
#pragma unroll
        for (int v = 0; v < 3; ++v)
          *reinterpret_cast<float4*>(wk + 4 * v) = reinterpret_cast<const float4*>(sm.w2 + co * 12)[v];
#pragma unroll
        for (int k = 0; k < 9; ++k) {
          const float w2v = wk[k];
          st[0][k] = fmaf(o[0][e], w2v, st[0][k]);
          st[1][k] = fmaf(o[1][e], w2v, st[1][k]);
        }
      }
#pragma unroll
      for (int p = 0; p < 2; ++p) {
        float v0 = o[p][0], v1 = o[p][1];
        const uint32_t hi = bf16x2_split(v0, v1);
        const uint32_t lo = bf16x2_split(v0, v1);
        sm.occ_hi[(pix0 + p) * kPixW + cp] = hi;
        sm.occ_lo[(pix0 + p) * kPixW + cp] = lo;
      }
    }
#pragma unroll
    for (int p = 0; p < 2; ++p)
#pragma unroll
      for (int k = 0; k < 9; ++k) sm.stap[k * kTapW + (y + 1) * (kG + 2) + (x0 + p + 1)] = st[p][k];
  }
  __syncthreads();

  // ---- phase C: hid2 = b2 + sum over taps of the neighbours' per-tap dot products; softmax,
  // arg-max of the probabilities (lowest index on ties), radius-5 soft arg-max (utils.py:116-150)
  float heat[2];
  {
    const float b2 = w.hid2_b[0];
#pragma unroll
    for (int p = 0; p < 2; ++p) {
      float a = b2;
#pragma unroll
      for (int ky = 0; ky < 3; ++ky)
#pragma unroll
        for (int kx = 0; kx < 3; ++kx)
          a += sm.stap[(ky * 3 + kx) * kTapW + (y + ky) * (kG + 2) + (x0 + p + kx)];
      heat[p] = a * temperature;
    }
  }
  int dummy;
  float gmax;
  block_max_first(fmaxf(heat[0], heat[1]), 0, sm.slot[0], &gmax, &dummy);
  float e[2];
  e[0] = expf(heat[0] - gmax);
  e[1] = expf(heat[1] - gmax);
  float gsum, u1, u2;
  block_sum3(e[0] + e[1], 0.f, 0.f, sm.slot[1], &gsum, &u1, &u2);
  float prob[2];
  float pbest = -1.f;
  int ibest = 0;
#pragma unroll
  for (int p = 0; p < 2; ++p) {
    prob[p] = e[p] / gsum;
    if (prob[p] > pbest) { pbest = prob[p]; ibest = y * kG + x0 + p; }
  }
  float pm;
  int am;
  block_max_first(pbest, ibest, sm.slot[2], &pm, &am);
  const float cx = (float)(am & 31) + 0.5f, cy = (float)(am >> 5) + 0.5f;
  float sx = 0.f, sy = 0.f, sw = 0.f;
#pragma unroll
  for (int p = 0; p < 2; ++p) {
    const float px = (float)(x0 + p) + 0.5f, py = (float)y + 0.5f;
    const float dx = px - cx, dy = py - cy;
    if (dx * dx + dy * dy < 25.f) { sx += px * prob[p]; sy += py * prob[p]; sw += prob[p]; }
  }
  float tx, ty, tw;
  block_sum3(sx, sy, sw, sm.slot[3], &tx, &ty, &tw);

  // ---- phase D: hid3 (pad(0,2,0,2), conv3x3 stride 2, 16->32) on the tensor cores.
  // warp = output row oy (16 output pixels = one m16 tile), 4 n8 tiles, one k16 step per tap.
  {
    const int oy = warp, g = lane >> 2, tq = lane & 3;
    float acc[4][4];
#pragma unroll
    for (int nt = 0; nt < 4; ++nt)
#pragma unroll
      for (int k = 0; k < 4; ++k) acc[nt][k] = 0.f;
#pragma unroll 1
    for (int tap = 0; tap < 9; ++tap) {
      const int ky = tap / 3, kx = tap - ky * 3;
      const int pa = ((2 * oy + ky + 1) * kOccW + (2 * g + kx + 1)) * kPixW;  // output pixel ox = g
      const int pb = pa + 16 * kPixW;                                         // ox = g + 8
      uint32_t ah[4], al[4];
      ah[0] = sm.occ_hi[pa + tq]; ah[1] = sm.occ_hi[pb + tq];
      ah[2] = sm.occ_hi[pa + tq + 4]; ah[3] = sm.occ_hi[pb + tq + 4];
      al[0] = sm.occ_lo[pa + tq]; al[1] = sm.occ_lo[pb + tq];
      al[2] = sm.occ_lo[pa + tq + 4]; al[3] = sm.occ_lo[pb + tq + 4];
#pragma unroll
      for (int nt = 0; nt < 4; ++nt) {
        const int wb = (tap * 32 + nt * 8 + g) * kW3Stride + tq;
        uint32_t bh[2] = {sm.w3_hi[wb], sm.w3_hi[wb + 4]};
        uint32_t bl[2] = {sm.w3_lo[wb], sm.w3_lo[wb + 4]};
        mma_bf16_16816(acc[nt], al, bh);
        mma_bf16_16816(acc[nt], ah, bl);
        mma_bf16_16816(acc[nt], ah, bh);
      }
    }
    // bias + ReLU, then the spatial sum of this warp's 16 pixels per channel: a thread owns
    // rows g, g+8 and channels nt*8 + 2*tq + {0,1}
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) {
#pragma unroll
      for (int e2 = 0; e2 < 2; ++e2) {
        const float b = sm.b3[nt * 8 + 2 * tq + e2];
        float v = fmaxf(acc[nt][e2] + b, 0.f) + fmaxf(acc[nt][2 + e2] + b, 0.f);
        v += __shfl_xor_sync(0xffffffffu, v, 4);
        v += __shfl_xor_sync(0xffffffffu, v, 8);
        v += __shfl_xor_sync(0xffffffffu, v, 16);
        if (g == 0) sm.mean32[warp][nt * 8 + 2 * tq + e2] = v;
      }
    }
  }
  __syncthreads();
  // The rest of the map (channel means, 32 -> 16 -> 2 MLP, outputs) is a few hundred FLOPs: warp 0
  // does it alone with shuffles while the other 15 warps already stage the next map (the mean32
  // rows are rewritten only in the next map's phase D, four barriers from here).
  if (warp == 0) {
    float m = 0.f;
#pragma unroll
    for (int k = 0; k < 16; ++k) m += sm.mean32[k][lane];
    head_tail(m * (1.0f / 256.0f), sm.w4, sm.b4, sm.w5, sm.b5, tx, ty, tw, am, kG, kG, n, t, T, query_tyx,
              init_h, init_w, points, occ_out, expd_out, argmax_out);
  }
  }  // map loop
}


// ------------------------------------------------------------------------ a6 head, any map size
// initial_resolution != (256, 256) (constructor argument, tapir_model.py:86) gives a cost map that
// is not 32 x 32.  The same head as the tensor-core kernel's for a gh x gw map: one CTA per map,
// ReLU(hid1) and the heat map staged in a per-CTA slice of the caller's workspace (L2 resident).
// A correctness path (every published checkpoint / demo uses 256 x 256), not a tuned one.
__global__ void __launch_bounds__(256) cost_volume_head_generic_kernel(
    const tapir_head_weights w, const float* __restrict__ cost_volume, int T, int num_maps, int gh,
    int gw, const float* __restrict__ query_tyx, float temperature, int init_h, int init_w,
    float* __restrict__ scratch, float* __restrict__ points, float* __restrict__ occ_out,
    float* __restrict__ expd_out, int* __restrict__ argmax_out) {
  __shared__ float w1s[16 * 9], b1s[16], w2s[16 * 9], w3s[32 * 16 * 9], b3s[32];
  __shared__ float mean32[8][32];  // [warp][channel] sums of ReLU(hid3)
  // one slot per block reduction of a map (4 per map): a slot is written again only in the next
  // map, and the map loop starts with __syncthreads(), so that write comes after every read
  __shared__ RedSlot<8> slot[4];
  const int tid = threadIdx.x;
  const int warp = tid >> 5, lane = tid & 31;
  const int pw = gw + 3, ph = gh + 3;  // index -1 .. size+1 (1 halo before, 2 after)
  const int plane = pw * ph;
  const int cells = gh * gw;
  float* occ = scratch + (size_t)blockIdx.x * (16 * plane + cells);  // [16][ph][pw]
  float* heat = occ + 16 * plane;                                    // [gh][gw]
  for (int i = tid; i < 16 * 9; i += 256) { w1s[i] = w.hid1_w[i]; w2s[i] = w.hid2_w[i]; }
  for (int i = tid; i < 32 * 16 * 9; i += 256) w3s[i] = w.hid3_w[i];
  if (tid < 16) b1s[tid] = w.hid1_b[tid];
  if (tid < 32) b3s[tid] = w.hid3_b[tid];
  for (int i = tid; i < 16 * plane; i += 256) occ[i] = 0.f;  // halos stay zero for every map
  const float b2 = w.hid2_b[0];
  const int oh = (gh - 1) / 2 + 1, ow = (gw - 1) / 2 + 1;  // pad (0,2,0,2), 3x3, stride 2, no padding
  for (int map = blockIdx.x; map < num_maps; map += gridDim.x) {
    const int n = map / T, t = map - n * T;
    const float* cv = cost_volume + (size_t)map * cells;
    __syncthreads();
    // hid1: conv3x3 1 -> 16, padding 1, ReLU
    for (int i = tid; i < cells; i += 256) {
      const int y = i / gw, x = i - y * gw;
      float win[9];
#pragma unroll
      for (int ky = 0; ky < 3; ++ky)
#pragma unroll
        for (int kx = 0; kx < 3; ++kx) {
          const int yy = y + ky - 1, xx = x + kx - 1;
          win[ky * 3 + kx] = (yy >= 0 && yy < gh && xx >= 0 && xx < gw) ? cv[yy * gw + xx] : 0.f;
        }
      for (int co = 0; co < 16; ++co) {
        float a = b1s[co];
#pragma unroll
        for (int k = 0; k < 9; ++k) a = fmaf(win[k], w1s[co * 9 + k], a);
        occ[co * plane + (y + 1) * pw + (x + 1)] = fmaxf(a, 0.f);
      }
    }
    __syncthreads();
    // hid2: conv3x3 16 -> 1, padding 1, x temperature; running maximum
    float lmax = -FLT_MAX;
    for (int i = tid; i < cells; i += 256) {
      const int y = i / gw, x = i - y * gw;
      float a = b2;
      for (int ci = 0; ci < 16; ++ci)
#pragma unroll
        for (int ky = 0; ky < 3; ++ky)
#pragma unroll
          for (int kx = 0; kx < 3; ++kx)
            a = fmaf(occ[ci * plane + (y + ky) * pw + (x + kx)], w2s[ci * 9 + ky * 3 + kx], a);
      const float h = a * temperature;
      heat[i] = h;
      lmax = fmaxf(lmax, h);
    }
    int dummy;
    float gmax;
    block_max_first(lmax, 0, slot[0], &gmax, &dummy);
    float lsum = 0.f;
    for (int i = tid; i < cells; i += 256) lsum += expf(heat[i] - gmax);
    float gsum, u1, u2;
    block_sum3(lsum, 0.f, 0.f, slot[1], &gsum, &u1, &u2);
    float pbest = -1.f;
    int ibest = 0;
    for (int i = tid; i < cells; i += 256) {  // ascending i: the first maximum is kept
      const float pr = expf(heat[i] - gmax) / gsum;
      if (pr > pbest) { pbest = pr; ibest = i; }
    }
    float pm;
    int am;
    block_max_first(pbest, ibest, slot[2], &pm, &am);
    const float cx = (float)(am % gw) + 0.5f, cy = (float)(am / gw) + 0.5f;
    float sx = 0.f, sy = 0.f, sw = 0.f;
    for (int i = tid; i < cells; i += 256) {
      const int y = i / gw, x = i - y * gw;
      const float px = (float)x + 0.5f, py = (float)y + 0.5f;
      const float dx = px - cx, dy = py - cy;
      if (dx * dx + dy * dy < 25.f) {
        const float pr = expf(heat[i] - gmax) / gsum;
        sx += px * pr; sy += py * pr; sw += pr;
      }
    }
    float tx, ty, tw;
    block_sum3(sx, sy, sw, slot[3], &tx, &ty, &tw);
    // hid3: conv3x3 stride 2 16 -> 32 on the (0,2,0,2)-padded activation, ReLU, spatial mean
    float msum[32];
#pragma unroll
    for (int c = 0; c < 32; ++c) msum[c] = 0.f;
    for (int o = tid; o < oh * ow; o += 256) {
      const int oy = o / ow, ox = o - oy * ow;
      float acc[32];
#pragma unroll
      for (int c = 0; c < 32; ++c) acc[c] = b3s[c];
      for (int ci = 0; ci < 16; ++ci)
#pragma unroll
        for (int ky = 0; ky < 3; ++ky)
#pragma unroll
          for (int kx = 0; kx < 3; ++kx) {
            const float v = occ[ci * plane + (2 * oy + ky + 1) * pw + (2 * ox + kx + 1)];
#pragma unroll
            for (int c = 0; c < 32; ++c) acc[c] = fmaf(v, w3s[(c * 16 + ci) * 9 + ky * 3 + kx], acc[c]);
          }
#pragma unroll
      for (int c = 0; c < 32; ++c) msum[c] += fmaxf(acc[c], 0.f);
    }
#pragma unroll
    for (int c = 0; c < 32; ++c) {
      const float v = warp_sum(msum[c]);
      if (lane == 0) mean32[warp][c] = v;
    }
    __syncthreads();
    // the MLP reads its 2.2 KB of weights through L1 rather than staging them in shared memory
    if (warp == 0) {
      float m = 0.f;
      for (int k = 0; k < 8; ++k) m += mean32[k][lane];
      head_tail(m / (float)(oh * ow), w.hid4_w, w.hid4_b, w.occ_w, w.occ_b, tx, ty, tw, am, gh, gw, n, t, T,
                query_tyx, init_h, init_w, points, occ_out, expd_out, argmax_out);
    }
  }
}

}  // namespace

int sample_query_features(const float* grid, int T, int gh, int gw, int C, const float* query_tyx,
                          int N, int vT, int vH, int vW, const int* frame_slot, float* out,
                          cudaStream_t s) {
  TAPIR_CHECK_ARG(grid && query_tyx && out && N > 0 && T > 0 && gh > 0 && gw > 0 && C > 0,
                  "sample_query_features: bad arguments");
  ProfileScope ps("sample_query", s, 0.0, (double)N * C * 4 * 9);
  // without a frame table the grid's own T normalises the time axis (the reference's call, where
  // the grid holds the whole clip); with one, the video's vT does
  sample_query_kernel<<<N, 128, 0, s>>>(grid, T, gh, gw, C, query_tyx, vT, vH, vW,
                                        frame_slot ? vT : T, frame_slot, out);
  count_launch();
  TAPIR_LAUNCH_CHECK("sample_query_kernel");
  return kOk;
}

int sample_query_rows(const tapir_query_grid* grids, int num_grids, int clips, int rows, int video_h,
                      int video_w, const int32_t* video_hw, const int32_t* count,
                      const tapir_query_request* requests, float* const* state, int num_state,
                      cudaStream_t s) {
  QueryRowsParams p = {};
  for (int i = 0; i < num_grids; ++i) p.grids[i] = grids[i];
  p.num_grids = num_grids;
  p.clips = clips;
  p.rows = rows;
  p.video_h = video_h;
  p.video_w = video_w;
  p.video_hw = video_hw;
  p.count = count;
  p.req = requests;
  p.state = state;
  // at most 32 CTAs per table entry: a launch without requests stays a few microseconds
  const dim3 grid((unsigned)(rows < 32 ? rows : 32), 1u + (unsigned)num_state);
  sample_query_rows_kernel<<<grid, 128, 0, s>>>(p);
  count_launch();
  TAPIR_LAUNCH_CHECK("sample_query_rows_kernel");
  return kOk;
}

namespace {
constexpr int kCvPlanes = 3;
struct CvPlan {
  __nv_bfloat16* q;
  __nv_bfloat16* g;
  float* cv;
  float* generic_scratch;  // maps other than 32 x 32 only
  int generic_ctas;
};
constexpr int kGenericCtasPerSm = 4;
// B clips of T frames with Q queries in all
size_t plan_cv(Arena& a, int B, long long Q, int T, int gh, int gw, int C, CvPlan* p) {
  const long long cells = (long long)T * gh * gw;
  p->q = a.take<__nv_bfloat16>((size_t)Q * C * kCvPlanes);
  p->g = a.take<__nv_bfloat16>((size_t)B * cells * C * kCvPlanes);
  p->cv = a.take<float>((size_t)Q * cells);
  p->generic_scratch = nullptr;
  p->generic_ctas = 0;
  if (gh != kG || gw != kG) {
    const long long maps = Q * T;
    const long long cap = 132ll * kGenericCtasPerSm;  // independent of the device: sizes must agree
    p->generic_ctas = (int)(maps < cap ? maps : cap);
    p->generic_scratch =
        a.take<float>((size_t)p->generic_ctas * (16 * (size_t)(gh + 3) * (gw + 3) + (size_t)gh * gw));
  }
  return a.off;
}
// B clips of N queries each (counts == nullptr) or of counts[b] queries; their T frames of
// cost maps.  One batched or grouped GEMM, then one head launch over the flattened queries.
int run_cost_volume(const tapir_head_weights* w, const float* qfeat, const float* grid, int B, int N,
                    const int* counts, int T, int gh, int gw, int C, const float* query_tyx,
                    float temperature, int init_h, int init_w, float* points, float* occ, float* expd,
                    int* argmax, void* ws, size_t ws_bytes, cudaStream_t s) {
  TAPIR_CHECK_ARG(w && qfeat && grid && points && occ && expd, "cost_volume_tracks: null pointer");
  TAPIR_CHECK_ARG(B > 0 && (counts == nullptr || B <= kGemmMaxGroups), "cost_volume_tracks: bad clip count B=%d", B);
  long long Q = (long long)B * N;
  if (counts != nullptr) {
    Q = 0;
    for (int b = 0; b < B; ++b) {
      TAPIR_CHECK_ARG(counts[b] > 0, "cost_volume_tracks: clip %d has %d queries", b, counts[b]);
      Q += counts[b];
    }
  }
  TAPIR_CHECK_ARG((counts != nullptr || N > 0) && T > 0 && C % 64 == 0,
                  "cost_volume_tracks: bad shape N=%d T=%d C=%d", N, T, C);
  TAPIR_CHECK_ARG(gh >= 2 && gw >= 2, "cost_volume_tracks: map %dx%d too small", gh, gw);
  // the documented per-call query limit for 32 x 32 maps (tapir_cost_volume_tracks_batched), the
  // same as the mixer's that refines these tracks
  TAPIR_CHECK_ARG((gh != kG || gw != kG) || Q <= 65535,
                  "cost_volume_tracks: at most 65535 queries per call (%lld)", Q);
  TAPIR_CHECK_ARG(Q < (1ll << 31), "cost_volume_tracks: %lld queries", Q);
  Arena arena(ws, ws_bytes);
  CvPlan p;
  plan_cv(arena, B, Q, T, gh, gw, C, &p);
  if (!arena.ok) {
    set_error("cost_volume_tracks: workspace too small (%zu < %zu)", ws_bytes, arena.off);
    return kWorkspaceTooSmall;
  }
  // qfeat [Q][C] -> planes [3][Q][C]; grid [B][T][gh][gw][C] -> planes [3][B*cells][C]
  const long long cells = (long long)T * gh * gw;
  const int BN = (int)Q;
  TAPIR_RETURN_IF(split_planes(qfeat, C, p.q, C, (long long)BN * C, BN, C, C, kCvPlanes, s));
  TAPIR_RETURN_IF(split_planes(grid, C, p.g, C, B * cells * C, B * cells, C, C, kCvPlanes, s));
  GemmArgs g;
  g.planes = kCvPlanes;
  g.N = (int)cells;
  g.K = C;
  g.a = p.q; g.lda = C; g.a_plane_stride = (long long)BN * C;
  g.b = p.g; g.ldb = C; g.b_plane_stride = B * cells * C;
  g.out_f32 = p.cv; g.ldo = (int)cells;
  g.b_batch_rows = cells;
  if (counts == nullptr) {
    // one batched GEMM: cv [B*N][cells], clip b = queries b*N.. against cells b*cells..
    g.M = N;
    g.batch = B;
    g.a_batch_rows = N;
    g.out_batch_stride = (long long)N * cells;
  } else {
    // one grouped GEMM: cv [Q][cells], clip b = its queries against cells b*cells..
    g.M = BN;
    g.groups = B;
    for (int b = 0; b < B; ++b) g.group_row0[b + 1] = g.group_row0[b] + counts[b];
  }
  g.tag = "cost_volume.gemm";
  TAPIR_RETURN_IF(gemm(g, s));
  // the heads index maps and query_tyx by flattened query b*N + n
  const int maps = BN * T;
  if (gh == kG && gw == kG) {
    static PerDeviceOnce configured;
    if (configured.pending()) {
      TAPIR_CUDA(cudaFuncSetAttribute(cost_volume_head_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      (int)sizeof(HeadTcSmem)));
      configured.mark();
    }
    // SURVEY.md 8(d): head = 2,950,208 FLOP per (n,t); 4 KB map in, 16 B out
    ProfileScope ps("cost_volume.head", s, 2950208.0 * BN * T, (double)BN * T * (4096 + 16));
    const int ctas = maps < num_sms() ? maps : num_sms();
    cost_volume_head_tc_kernel<<<ctas, kHT, sizeof(HeadTcSmem), s>>>(
        *w, p.cv, T, maps, query_tyx, temperature, init_h, init_w, points, occ, expd, argmax);
    count_launch();
    TAPIR_LAUNCH_CHECK("cost_volume_head_tc_kernel");
    return kOk;
  }
  // any other initial_resolution (tapir_model.py:86): generic-size head
  ProfileScope ps("cost_volume.head", s, 2950208.0 / 1024.0 * gh * gw * BN * T,
                  (double)BN * T * (4.0 * gh * gw + 16));
  cost_volume_head_generic_kernel<<<p.generic_ctas, 256, 0, s>>>(
      *w, p.cv, T, maps, gh, gw, query_tyx, temperature, init_h, init_w, p.generic_scratch, points, occ,
      expd, argmax);
  count_launch();
  TAPIR_LAUNCH_CHECK("cost_volume_head_generic_kernel");
  return kOk;
}
}  // namespace

size_t cost_volume_workspace_bytes(int B, long long Q, int T, int gh, int gw, int C) {
  if (B < 1 || Q < 0) return 0;
  Arena a(nullptr, 0);
  CvPlan p;
  return plan_cv(a, B, Q, T, gh, gw, C, &p) + 256;
}

int cost_volume_tracks(const tapir_head_weights* w, const float* qfeat, const float* grid, int B,
                       int N, int T, int gh, int gw, int C, const float* query_tyx, float temperature,
                       int init_h, int init_w, float* points, float* occ, float* expd, int* argmax,
                       void* ws, size_t ws_bytes, cudaStream_t s) {
  return run_cost_volume(w, qfeat, grid, B, N, nullptr, T, gh, gw, C, query_tyx, temperature, init_h,
                         init_w, points, occ, expd, argmax, ws, ws_bytes, s);
}

int cost_volume_tracks_ragged(const tapir_head_weights* w, const float* qfeat, const float* grid, int B,
                              const int* counts, int T, int gh, int gw, int C, const float* query_tyx,
                              float temperature, int init_h, int init_w, float* points, float* occ,
                              float* expd, int* argmax, void* ws, size_t ws_bytes, cudaStream_t s) {
  TAPIR_CHECK_ARG(counts != nullptr, "cost_volume_tracks_ragged: null counts");
  return run_cost_volume(w, qfeat, grid, B, 0, counts, T, gh, gw, C, query_tyx, temperature, init_h,
                         init_w, points, occ, expd, argmax, ws, ws_bytes, s);
}

}  // namespace tapir
