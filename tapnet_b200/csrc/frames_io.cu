// The callers either side of the hot path (SURVEY 8f rows 1 and 2), as HBM-bound one-pass kernels:
//   * frame ingest: uint8 camera / dataset frames -> centre crop -> bilinear resize -> [-1,1]
//     (pytorch_live_demo.py:30-41 preprocess_frames, :88-95 get_frame, utils.py:26-42 bilinear)
//   * output post-processing: visibility flag (pytorch_live_demo.py:57-59,
//     utils/model_utils.py:376-389) and the TAP-Vid metric counters
//     (tapvid/evaluation_datasets.py:48-192) without leaving the device.
#include "kernels.cuh"

namespace tapir {
namespace {

int grid_for(long long total, int block = 256) {
  long long g = ceil_div_ll(total, block);
  const long long cap = (long long)num_sms() * 16;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return (int)g;
}

// preprocess_frames: x / 255 * 2 - 1 in fp32, every operation rounded (no FMA contraction)
__device__ __forceinline__ float normalise_u8(uint8_t v) {
  return __fsub_rn(__fmul_rn(__fdiv_rn((float)v, 255.f), 2.f), 1.f);
}

// The 256 possible inputs of normalise_u8, tabulated once per CTA (the IEEE division is ~10
// instructions; the table makes the kernels pure load/store streams).
__device__ __forceinline__ void fill_lut(float* lut) {
  for (int i = threadIdx.x; i < 256; i += blockDim.x) lut[i] = normalise_u8((uint8_t)i);
  __syncthreads();
}

// preprocess_frames alone (no crop, no resize): 4 bytes in, one float4 out per thread and trip,
// both fully coalesced.
__global__ void __launch_bounds__(256) preprocess_u8_kernel(const uint8_t* __restrict__ src,
                                                            float* __restrict__ dst, long long n) {
  __shared__ float lut[256];
  fill_lut(lut);
  const long long n4 = n >> 2;
  const long long stride = (long long)gridDim.x * blockDim.x;
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
#pragma unroll 4
  for (; i < n4; i += stride) {
    const uchar4 v = reinterpret_cast<const uchar4*>(src)[i];
    reinterpret_cast<float4*>(dst)[i] = make_float4(lut[v.x], lut[v.y], lut[v.z], lut[v.w]);
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) dst[(n4 << 2) + threadIdx.x] = lut[src[(n4 << 2) + threadIdx.x]];
}

// uint8 RGB pixel (y, x) of the crop window at (cy, cx) of frame f of an H x W frame.
struct RgbWindow {
  const uint8_t* __restrict__ src;
  int H, W, cy, cx;
  __device__ __forceinline__ void pixel(long long f, int y, int x, uint8_t (&rgb)[3]) const {
    const uint8_t* p = src + (f * H + cy) * (long long)W * 3 + (long long)cx * 3 + ((long long)y * W + x) * 3;
    rgb[0] = p[0];
    rgb[1] = p[1];
    rgb[2] = p[2];
  }
};

// One ch x cw window of uint8 RGB pixels for every frame of the launch (RgbWindow or
// Yuv420Reader), as ingest_frames_kernel reads it: each tap normalised through the table.
template <typename Reader>
struct U8Frames {
  Reader r;
  int ch, cw;
  __device__ __forceinline__ void window(long long, int& h, int& w) const { h = ch; w = cw; }
  __device__ __forceinline__ bool copies(long long, int oH, int oW) const { return ch == oH && cw == oW; }
  __device__ __forceinline__ void tap(const float* lut, long long f, int y, int x, float (&v)[3]) const {
    uint8_t p[3];
    r.pixel(f, y, x, p);
    v[0] = lut[p[0]];
    v[1] = lut[p[1]];
    v[2] = lut[p[2]];
  }
};

// Device form of one tapir_ingest_desc (checked by the entry point).
struct IngestFrame {
  Yuv420Reader yuv;  // TAPIR_INGEST_YUV420: frame 0 of it
  const uint8_t* src;  // TAPIR_INGEST_U8: pixel (y0, x0) of the window
  long long pitch;     // TAPIR_INGEST_U8: row pitch in bytes
  int format, h, w;  // window size
};

// Up to TAPIR_INGEST_MAX_FRAMES frames of their own format and window, one descriptor each.
struct DescFrames {
  IngestFrame fr[TAPIR_INGEST_MAX_FRAMES];
  __device__ __forceinline__ void window(long long f, int& h, int& w) const { h = fr[f].h; w = fr[f].w; }
  __device__ __forceinline__ bool copies(long long f, int oH, int oW) const {
    return fr[f].h == oH && fr[f].w == oW;
  }
  __device__ __forceinline__ void tap(const float* lut, long long f, int y, int x, float (&v)[3]) const {
    const IngestFrame& d = fr[f];
    uint8_t p[3];
    if (d.format == TAPIR_INGEST_U8) {
      const uint8_t* q = d.src + (long long)y * d.pitch + (long long)x * 3;
      p[0] = q[0];
      p[1] = q[1];
      p[2] = q[2];
    } else {
      d.yuv.pixel(0, y, x, p);
    }
    v[0] = lut[p[0]];
    v[1] = lut[p[1]];
    v[2] = lut[p[2]];
  }
};

// crop + normalise + resize.  A CTA walks over runs of 256 consecutive output pixels: one thread
// computes one pixel (3 channels) into shared memory, then the run's 768 floats leave as float4
// rows (the direct 12-byte-strided stores would touch every sector three times).  The resize is
// F.interpolate(mode='bilinear', align_corners=False) of the normalised crop, i.e. the same
// arithmetic as bilinear_resize_kernel (backbone.cu) applied after normalise_u8.  Src gives each
// frame's window size and its normalised pixels (U8Frames of RgbWindow or Yuv420Reader converting
// each tap, or DescFrames with one window and format per frame).  The source is a grid constant:
// DescFrames' table is indexed by frame without a local copy.
template <typename Src>
__global__ void __launch_bounds__(256) ingest_frames_kernel(const __grid_constant__ Src src,
                                                            float* __restrict__ dst, int oH, int oW,
                                                            long long total, bool dst_aligned16) {
  __shared__ float lut[256];
  __shared__ __align__(16) float stage[256 * 3];
  fill_lut(lut);
  for (long long i0 = blockIdx.x * 256LL; i0 < total; i0 += (long long)gridDim.x * 256) {
    const long long i = i0 + threadIdx.x;
    if (i < total) {
      int ox, oy;
      long long f;
      if (total <= 0x7fffffffLL) {  // 32-bit divisions (the 64-bit ones cost more than the loads)
        const unsigned u = (unsigned)i, r = u / (unsigned)oW;
        ox = (int)(u - r * (unsigned)oW);
        const unsigned q = r / (unsigned)oH;
        oy = (int)(r - q * (unsigned)oH);
        f = q;
      } else {
        ox = (int)(i % oW);
        const long long r = i / oW;
        oy = (int)(r % oH);
        f = r / oH;
      }
      int ch, cw;
      src.window(f, ch, cw);
      float* o = stage + threadIdx.x * 3;
      if (src.copies(f, oH, oW)) {
        float v[3];
        src.tap(lut, f, oy, ox, v);
        o[0] = v[0];
        o[1] = v[1];
        o[2] = v[2];
      } else {
        const float sy = (float)ch / (float)oH, sx = (float)cw / (float)oW;
        float fy = sy * (oy + 0.5f) - 0.5f;
        float fx = sx * (ox + 0.5f) - 0.5f;
        if (fy < 0.f) fy = 0.f;
        if (fx < 0.f) fx = 0.f;
        const int y0 = (int)fy, x0 = (int)fx;
        const int y1 = y0 + ((y0 < ch - 1) ? 1 : 0), x1 = x0 + ((x0 < cw - 1) ? 1 : 0);
        const float ly = fy - y0, lx = fx - x0;
        const float hy = 1.f - ly, hx = 1.f - lx;
        float v00[3], v01[3], v10[3], v11[3];
        src.tap(lut, f, y0, x0, v00);
        src.tap(lut, f, y0, x1, v01);
        src.tap(lut, f, y1, x0, v10);
        src.tap(lut, f, y1, x1, v11);
#pragma unroll
        for (int c = 0; c < 3; ++c)
          o[c] = hy * (hx * v00[c] + lx * v01[c]) + ly * (hx * v10[c] + lx * v11[c]);
      }
    }
    __syncthreads();
    const long long left = total - i0;  // pixels in this run
    if (left >= 256 && dst_aligned16) {
      if (threadIdx.x < 192)  // i0 * 12 bytes is a multiple of 16: aligned float4 rows
        reinterpret_cast<float4*>(dst + i0 * 3)[threadIdx.x] = reinterpret_cast<const float4*>(stage)[threadIdx.x];
    } else {
      for (int e = threadIdx.x; e < (int)left * 3; e += 256) dst[i0 * 3 + e] = stage[e];
    }
    __syncthreads();
  }
}

// YUV 4:2:0 crop window -> dense uint8 RGB [frames][h][w][3]; one thread per pixel.
__global__ void __launch_bounds__(256) yuv420_to_rgb_kernel(const Yuv420Reader src, int h, int w,
                                                            uint8_t* __restrict__ dst,
                                                            long long total) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int x = (int)(i % w);
    const long long r = i / w;
    const int y = (int)(r % h);
    uint8_t p[3];
    src.pixel(r / h, y, x, p);
    dst[i * 3 + 0] = p[0];
    dst[i * 3 + 1] = p[1];
    dst[i * 3 + 2] = p[2];
  }
}

__device__ __forceinline__ float sigmoidf(float x) { return 1.f / (1.f + expf(-x)); }

// pytorch_live_demo.py:57-59: visible = (1 - sigmoid(occ)) * (1 - sigmoid(expd)) > 0.5
__device__ __forceinline__ bool visible_from_logits(float occ, float expd) {
  return __fmul_rn(1.f - sigmoidf(occ), 1.f - sigmoidf(expd)) > 0.5f;
}

__global__ void __launch_bounds__(256) postprocess_occlusions_kernel(const float* __restrict__ occ,
                                                                     const float* __restrict__ expd,
                                                                     long long n,
                                                                     uint8_t* __restrict__ visible) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x)
    visible[i] = visible_from_logits(occ[i], expd[i]) ? 1 : 0;
}

// tapvid/evaluation_datasets.py:48-192.  One warp per track (b, n); the 18 integer counters of a
// track are exact, the ratios are formed by the host from their sums (per video or per track).
//   [0] evaluated frames            [1] occlusion prediction == ground truth
//   [2] ground-truth visible        [3+i] within threshold 2^i and visible (i = 0..4)
//   [8+i] true positives            [13+i] false positives
__global__ void __launch_bounds__(256) tapvid_counts_kernel(const tapir_tapvid_args a) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  const int tracks = a.B * a.N;
  if (warp >= tracks) return;
  const int T = a.T;
  // evaluation_datasets.py:125-127: np.round (half to even) then int32
  const int qf = __float2int_rn(a.query_points[(long long)warp * 3]);
  const long long base = (long long)warp * T;
  int cnt[TAPIR_TAPVID_COUNTERS];
#pragma unroll
  for (int k = 0; k < TAPIR_TAPVID_COUNTERS; ++k) cnt[k] = 0;
  for (int t = lane; t < T; t += 32) {
    // :116-123: 'first' evaluates frames after the query frame, 'strided' all but the query frame
    const bool eval = (a.query_mode == 0) ? (t > qf) : (t != qf);
    if (!eval) continue;
    const bool gt_occ = a.gt_occluded[base + t] != 0;
    bool pred_occ;
    if (a.pred_occluded != nullptr)
      pred_occ = a.pred_occluded[base + t] != 0;
    else
      pred_occ = !visible_from_logits(a.pred_occ_logits[base + t], a.pred_expd_logits[base + t]);
    const float dx = __fsub_rn(a.pred_tracks[(base + t) * 2 + 0], a.gt_tracks[(base + t) * 2 + 0]);
    const float dy = __fsub_rn(a.pred_tracks[(base + t) * 2 + 1], a.gt_tracks[(base + t) * 2 + 1]);
    const float d2 = __fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy));  // :148-151
    const bool vis = !gt_occ, pvis = !pred_occ;
    cnt[0] += 1;
    cnt[1] += (pred_occ == gt_occ);
    cnt[2] += vis;
#pragma unroll
    for (int i = 0; i < 5; ++i) {
      const float th = (float)(1 << i);
      const bool within = d2 < th * th;
      const bool correct = within && vis;
      cnt[3 + i] += correct;
      cnt[8 + i] += correct && pvis;
      cnt[13 + i] += ((!vis) && pvis) || ((!within) && pvis);  // :177-179
    }
  }
#pragma unroll
  for (int k = 0; k < TAPIR_TAPVID_COUNTERS; ++k) {
    int v = cnt[k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0) a.counts[(long long)warp * TAPIR_TAPVID_COUNTERS + k] = v;
  }
}

// aj_rd.py calculate_jaccard_for_segment's ratio: float32(TP) / float32(gt_pos + FP), 0 / 0 -> nan
__device__ __forceinline__ float jaccard_ratio(int tp, int den) {
  return den == 0 ? __int_as_float(0x7fc00000) : __fdiv_rn(__int2float_rn(tp), __int2float_rn(den));
}

// tapnextpp/metrics/aj_rd.py compute_raw_redetection_stats.  One warp per track (b, n); lane i
// holds frame c0 + i of each 32-frame chunk.
//   pass 1, forward over gt_visible only: the reappearances, their durations (distance to the
//     last visible frame, from a ballot), eligibility against the running maximum of the earlier
//     durations (a max scan, only in chunks that hold a reappearance), compacted in t order into
//     the track's slots.
//   pass 2, backward from the last frame to the first event: suffix counts of gt-visible and of
//     TP / FP per threshold (ballot + popc, carried across chunks), read off by the lanes that
//     hold an event frame; the events of a chunk come back from pass 1's slots.
// Frames before the first eligible event are read once, the others twice (gt_visible) or once.
__global__ void __launch_bounds__(256) redetection_events_kernel(const tapir_redetection_args a, int K) {
  constexpr unsigned kAll = 0xffffffffu;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= a.B * a.N) return;
  const int T = a.T;
  const long long base = (long long)warp * T, slot0 = (long long)warp * K;
  const unsigned below = (1u << lane) - 1u, from_me = ~below;

  int last_vis = -1, max_d = -1, count = 0;
  bool prev_vis = false;
  for (int c0 = 0; c0 < T; c0 += 32) {
    const int t = c0 + lane;
    const bool g = t < T && a.gt_visible[base + t] != 0;
    const unsigned vis = __ballot_sync(kAll, g);
    const bool g_prev = lane == 0 ? prev_vis : ((vis >> (lane - 1)) & 1u) != 0;
    const bool event = g && !g_prev && t >= 1;
    if (__ballot_sync(kAll, event) != 0) {
      // count_consecutive_invisibility at t: frames since the last visible one before t
      const unsigned vb = vis & below;
      const int d = t - 1 - (vb != 0 ? c0 + 31 - __clz(vb) : last_vis);
      int m = event ? d : -1;  // inclusive max scan of the chunk's durations
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(kAll, m, o);
        if (lane >= o) m = max(m, v);
      }
      int earlier = __shfl_up_sync(kAll, m, 1);
      earlier = max(lane == 0 ? -1 : earlier, max_d);
      const bool eligible = event && d > earlier;  // strictly longer than every earlier event
      const unsigned em = __ballot_sync(kAll, eligible);
      if (eligible) {
        const long long s = slot0 + count + __popc(em & below);
        a.event_t[s] = t;
        a.event_duration[s] = d;
      }
      count += __popc(em);
      max_d = max(max_d, __shfl_sync(kAll, m, 31));
    }
    if (vis != 0) last_vis = c0 + 31 - __clz(vis);
    prev_vis = (vis >> 31) != 0;
  }
  if (lane == 0) a.event_count[warp] = count;
  if (count == 0) return;
  __syncwarp();  // the slots written above, visible to every lane

  const int nd = a.num_thresholds;
  int gt_pos = 0, tp[TAPIR_REDETECTION_MAX_THRESHOLDS], fp[TAPIR_REDETECTION_MAX_THRESHOLDS];
#pragma unroll
  for (int j = 0; j < TAPIR_REDETECTION_MAX_THRESHOLDS; ++j) tp[j] = fp[j] = 0;
  int k = count - 1;  // the latest event not yet read off
  int next_t = a.event_t[slot0 + k];
  const int first_t = a.event_t[slot0];
  for (int c0 = (T - 1) & ~31; c0 + 31 >= first_t; c0 -= 32) {
    const int t = c0 + lane;
    bool g = false, p = false;
    float dx = 0.f, dy = 0.f;
    if (t < T) {
      const long long i = base + t;
      g = a.gt_visible[i] != 0;
      p = a.pred_visible != nullptr ? a.pred_visible[i] != 0
                                    : visible_from_logits(a.pred_occ_logits[i], a.pred_expd_logits[i]);
      dx = __fsub_rn(a.pred_tracks[2 * i], a.gt_tracks[2 * i]);
      dy = __fsub_rn(a.pred_tracks[2 * i + 1], a.gt_tracks[2 * i + 1]);
    }
    // torch.linalg.norm(., dim=-1) of a float32 pair on the CPU: dx * dx rounded, one FMA, sqrt
    const float dist = __fsqrt_rn(__fmaf_rn(dy, dy, __fmul_rn(dx, dx)));
    unsigned ev_bits = 0;  // the chunk's event frames
    const int k_last = k;
    while (k >= 0 && next_t >= c0) {
      ev_bits |= 1u << (next_t - c0);
      --k;
      next_t = k >= 0 ? a.event_t[slot0 + k] : -1;
    }
    const bool at_event = ((ev_bits >> lane) & 1u) != 0;
    float* out = a.event_values + (slot0 + k_last - (__popc(ev_bits >> lane) - 1)) * nd;
    const unsigned gm = __ballot_sync(kAll, g);
    const int gt_here = gt_pos + __popc(gm & from_me);
#pragma unroll
    for (int j = 0; j < TAPIR_REDETECTION_MAX_THRESHOLDS; ++j) {
      if (j < nd) {
        const bool within = dist <= a.thresholds[j];  // false for a NaN distance
        const unsigned tpm = __ballot_sync(kAll, within && g && p);
        const unsigned fpm = __ballot_sync(kAll, p && (!g || !within));
        if (at_event)
          out[j] = jaccard_ratio(tp[j] + __popc(tpm & from_me), gt_here + fp[j] + __popc(fpm & from_me));
        tp[j] += __popc(tpm);
        fp[j] += __popc(fpm);
      }
    }
    gt_pos += __popc(gm);
  }
}

}  // namespace

int ingest_frames(const uint8_t* src, int frames, int H, int W, int crop_y, int crop_x, int crop_h,
                  int crop_w, float* dst, int oH, int oW, cudaStream_t s) {
  TAPIR_CHECK_ARG(src && dst && frames > 0 && H > 0 && W > 0 && oH > 0 && oW > 0,
                  "ingest_frames: bad arguments");
  TAPIR_CHECK_ARG(crop_y >= 0 && crop_x >= 0 && crop_h > 0 && crop_w > 0 && crop_y + crop_h <= H &&
                      crop_x + crop_w <= W,
                  "ingest_frames: crop (%d,%d,%d,%d) outside the %dx%d frame", crop_y, crop_x, crop_h,
                  crop_w, H, W);
  const long long total = (long long)frames * oH * oW;
  ProfileScope ps("ingest_frames", s, 0.0,
                  (double)frames * crop_h * crop_w * 3 + (double)total * 12);
  if (crop_y == 0 && crop_x == 0 && crop_h == H && crop_w == W && oH == H && oW == W &&
      (reinterpret_cast<uintptr_t>(src) & 3) == 0 && (reinterpret_cast<uintptr_t>(dst) & 15) == 0) {
    const long long n = total * 3;
    preprocess_u8_kernel<<<grid_for(n / 4 / 4 + 1), 256, 0, s>>>(src, dst, n);
  } else {
    ingest_frames_kernel<<<grid_for(total), 256, 0, s>>>(
        U8Frames<RgbWindow>{RgbWindow{src, H, W, crop_y, crop_x}, crop_h, crop_w}, dst, oH, oW, total,
        (reinterpret_cast<uintptr_t>(dst) & 15) == 0);
  }
  count_launch();
  TAPIR_LAUNCH_CHECK("ingest_frames_kernel");
  return kOk;
}

int ingest_frames_yuv420(const Yuv420Reader& src, int frames, int h, int w, float* dst, int oH,
                         int oW, cudaStream_t s) {
  TAPIR_CHECK_ARG(dst && frames > 0 && h > 0 && w > 0 && oH > 0 && oW > 0,
                  "ingest_frames_yuv420: bad arguments");
  const long long total = (long long)frames * oH * oW;
  ProfileScope ps("ingest_frames_yuv420", s, 0.0, (double)frames * h * w * 1.5 + (double)total * 12);
  ingest_frames_kernel<<<grid_for(total), 256, 0, s>>>(U8Frames<Yuv420Reader>{src, h, w}, dst, oH, oW,
                                                       total, (reinterpret_cast<uintptr_t>(dst) & 15) == 0);
  count_launch();
  TAPIR_LAUNCH_CHECK("ingest_frames_kernel");
  return kOk;
}

int ingest_frames_multi(const tapir_ingest_desc* descs, int frames, float* dst, int oH, int oW,
                        cudaStream_t s) {
  TAPIR_CHECK_ARG(descs && dst && frames > 0 && oH > 0 && oW > 0,
                  "ingest_frames_multi: bad arguments (descs %p, frames %d, dst %p, out %dx%d)",
                  (const void*)descs, frames, (void*)dst, oH, oW);
  TAPIR_CHECK_ARG((long long)frames * oH * oW * 3 < (1ll << 40), "ingest_frames_multi: output too large");
  // every descriptor first: nothing is launched unless all of them are good
  double in_bytes = 0;
  for (int i = 0; i < frames; ++i) {
    const tapir_ingest_desc& d = descs[i];
    if (d.format == TAPIR_INGEST_YUV420) {
      Yuv420Reader r;
      TAPIR_RETURN_IF(make_yuv420_reader(&d.yuv, 1, "ingest_frames_multi", &r));
      in_bytes += (double)d.yuv.h * d.yuv.w * 1.5;
      continue;
    }
    TAPIR_CHECK_ARG(d.format == TAPIR_INGEST_U8,
                    "ingest_frames_multi: frame %d: format %d is not 1 (uint8) or 2 (YUV 4:2:0)", i,
                    d.format);
    TAPIR_CHECK_ARG(d.src != nullptr && d.H > 0 && d.W > 0 && d.pitch >= 3ll * d.W,
                    "ingest_frames_multi: frame %d: src %p, %dx%d frame, row pitch %lld", i, d.src, d.H,
                    d.W, (long long)d.pitch);
    TAPIR_CHECK_ARG(d.y0 >= 0 && d.x0 >= 0 && d.h > 0 && d.w > 0 && (long long)d.y0 + d.h <= d.H &&
                        (long long)d.x0 + d.w <= d.W,
                    "ingest_frames_multi: frame %d: crop (%d,%d,%d,%d) outside the %dx%d frame", i, d.y0,
                    d.x0, d.h, d.w, d.H, d.W);
    in_bytes += (double)d.h * d.w * 3;
  }
  for (int f0 = 0; f0 < frames; f0 += TAPIR_INGEST_MAX_FRAMES) {
    const int n = frames - f0 < TAPIR_INGEST_MAX_FRAMES ? frames - f0 : TAPIR_INGEST_MAX_FRAMES;
    DescFrames src;
    for (int i = 0; i < n; ++i) {
      const tapir_ingest_desc& d = descs[f0 + i];
      IngestFrame& fr = src.fr[i];
      fr = IngestFrame{};
      fr.format = d.format;
      if (d.format == TAPIR_INGEST_YUV420) {
        make_yuv420_reader(&d.yuv, 1, "ingest_frames_multi", &fr.yuv);
        fr.h = d.yuv.h;
        fr.w = d.yuv.w;
      } else {
        fr.src = static_cast<const uint8_t*>(d.src) + (long long)d.y0 * d.pitch + (long long)d.x0 * 3;
        fr.pitch = d.pitch;
        fr.h = d.h;
        fr.w = d.w;
      }
    }
    float* out = dst + (long long)f0 * oH * oW * 3;
    const long long total = (long long)n * oH * oW;
    ProfileScope ps("ingest_frames_multi", s, 0.0, in_bytes * n / frames + (double)total * 12);
    ingest_frames_kernel<<<grid_for(total), 256, 0, s>>>(src, out, oH, oW, total,
                                                         (reinterpret_cast<uintptr_t>(out) & 15) == 0);
    count_launch();
    TAPIR_LAUNCH_CHECK("ingest_frames_kernel");
  }
  return kOk;
}

int yuv420_to_rgb(const Yuv420Reader& src, int frames, int h, int w, uint8_t* dst, cudaStream_t s) {
  TAPIR_CHECK_ARG(dst && frames > 0 && h > 0 && w > 0, "yuv420_to_rgb: bad arguments");
  const long long total = (long long)frames * h * w;
  ProfileScope ps("yuv420_to_rgb", s, 0.0, (double)total * 4.5);
  yuv420_to_rgb_kernel<<<grid_for(total), 256, 0, s>>>(src, h, w, dst, total);
  count_launch();
  TAPIR_LAUNCH_CHECK("yuv420_to_rgb_kernel");
  return kOk;
}

int postprocess_occlusions(const float* occ, const float* expd, long long n, uint8_t* visible,
                           cudaStream_t s) {
  TAPIR_CHECK_ARG(occ && expd && visible && n > 0, "postprocess_occlusions: bad arguments");
  ProfileScope ps("postprocess_occlusions", s, 0.0, (double)n * 9);
  postprocess_occlusions_kernel<<<grid_for(n), 256, 0, s>>>(occ, expd, n, visible);
  count_launch();
  TAPIR_LAUNCH_CHECK("postprocess_occlusions_kernel");
  return kOk;
}

int tapvid_counts(const tapir_tapvid_args* a, cudaStream_t s) {
  TAPIR_CHECK_ARG(a != nullptr && a->B > 0 && a->N > 0 && a->T > 0, "tapvid_counts: bad shape");
  TAPIR_CHECK_ARG(a->query_points && a->gt_occluded && a->gt_tracks && a->pred_tracks && a->counts,
                  "tapvid_counts: null pointer");
  TAPIR_CHECK_ARG(a->pred_occluded != nullptr || (a->pred_occ_logits && a->pred_expd_logits),
                  "tapvid_counts: need pred_occluded or both logit arrays");
  TAPIR_CHECK_ARG(a->query_mode == 0 || a->query_mode == 1,
                  "tapvid_counts: query_mode must be 0 ('first') or 1 ('strided')");
  const long long tracks = (long long)a->B * a->N;
  ProfileScope ps("tapvid_counts", s, 0.0, (double)tracks * a->T * 18);
  const int warps_per_block = 8;
  tapvid_counts_kernel<<<(unsigned)ceil_div_ll(tracks, warps_per_block), 32 * warps_per_block, 0, s>>>(*a);
  count_launch();
  TAPIR_LAUNCH_CHECK("tapvid_counts_kernel");
  return kOk;
}

int redetection_max_events(int T) {
  if (T < 1) return 0;
  long long k = (long long)((sqrt(9.0 + 8.0 * T) - 3.0) / 2.0);
  while (k > 0 && k * (k + 3) / 2 > T) --k;
  while ((k + 1) * (k + 4) / 2 <= T) ++k;
  return (int)k;
}

int redetection_events(const tapir_redetection_args* a, cudaStream_t s) {
  TAPIR_CHECK_ARG(a != nullptr, "redetection_events: null args");
  TAPIR_CHECK_ARG(a->B > 0 && a->N > 0 && a->T > 0 && a->T <= (1 << 30) &&
                      (long long)a->B * a->N <= (1ll << 26),
                  "redetection_events: bad shape B=%d N=%d T=%d", a->B, a->N, a->T);
  TAPIR_CHECK_ARG(a->num_thresholds >= 1 && a->num_thresholds <= TAPIR_REDETECTION_MAX_THRESHOLDS,
                  "redetection_events: num_thresholds=%d outside 1..%d", a->num_thresholds,
                  TAPIR_REDETECTION_MAX_THRESHOLDS);
  TAPIR_CHECK_ARG(a->gt_visible && a->pred_tracks && a->gt_tracks && a->event_count,
                  "redetection_events: null pointer");
  TAPIR_CHECK_ARG(a->pred_visible != nullptr || (a->pred_occ_logits && a->pred_expd_logits),
                  "redetection_events: need pred_visible or both logit arrays");
  const long long tracks = (long long)a->B * a->N;
  const int K = redetection_max_events(a->T);
  TAPIR_CHECK_ARG(K == 0 || (a->event_t && a->event_duration && a->event_values),
                  "redetection_events: null event array");
  TAPIR_CHECK_ARG(a->capacity >= tracks * K,
                  "redetection_events: capacity %lld < %lld slots (B N K(T), K(%d) = %d)",
                  (long long)a->capacity, tracks * K, a->T, K);
  const double pred_bytes = a->pred_visible != nullptr ? 1.0 : 8.0;
  ProfileScope ps("redetection_events", s, 0.0, (double)tracks * a->T * (1.0 + pred_bytes + 16.0));
  const int warps_per_block = 8;
  redetection_events_kernel<<<(unsigned)ceil_div_ll(tracks, warps_per_block), 32 * warps_per_block, 0,
                              s>>>(*a, K);
  count_launch();
  TAPIR_LAUNCH_CHECK("redetection_events_kernel");
  return kOk;
}

}  // namespace tapir
