// YUV -> uint8 RGB (the contract of tapir_yuv_frames in include/tapir_b200.h), shared by the stem
// conv's loader (backbone.cu) and the ingest / conversion kernels (frames_io.cu).  Integer
// arithmetic only, so every reader produces the same bytes.  One reader for every layout: the
// sample type (uint8_t / uint16_t) is a template parameter, the layout fields are read at run time.
#pragma once
#include "../../include/tapir_b200.h"
#include "common.cuh"

namespace tapir {

// A crop window of tapir_yuv_frames as the kernels read it: pixel<T>(f, r, c) is window pixel
// (r, c) of frame f, i.e. frame pixel (y0 + r, x0 + c).  Strides, pitches and steps in samples.
struct YuvLayout {
  const void* y;
  const void* u;
  const void* v;
  long long y_frame, u_frame, v_frame;
  long long y_pitch, u_pitch, v_pitch;
  int luma_step, chroma_step, shift_x, shift_y, y0, x0;
  int mask, shl;         // v16 = (s & mask) << shl
  int k, c_off;          // luma gain and 16-bit offset: (298, 4096) limited range, (256, 0) full
  int cr, gu, gv, bu;    // chroma coefficients (R from V, G from U and V, B from U)

#ifdef __CUDACC__
  __device__ __forceinline__ static int clamp255(int x) { return x < 0 ? 0 : (x > 255 ? 255 : x); }

  template <typename T>
  __device__ __forceinline__ void pixel(long long f, int r, int c, uint8_t (&rgb)[3]) const {
    const int ay = y0 + r, ax = x0 + c;
    const long long cy = ay >> shift_y, cx = (long long)(ax >> shift_x) * chroma_step;
    const T* py = static_cast<const T*>(y) + f * y_frame + ay * y_pitch + (long long)ax * luma_step;
    const T* pu = static_cast<const T*>(u) + f * u_frame + cy * u_pitch + cx;
    const T* pv = static_cast<const T*>(v) + f * v_frame + cy * v_pitch + cx;
    const int Y = ((int)__ldg(py) & mask) << shl;
    const int D = (((int)__ldg(pu) & mask) << shl) - 32768;
    const int E = (((int)__ldg(pv) & mask) << shl) - 32768;
    const int L = k * (Y - c_off) + 32768;
    rgb[0] = (uint8_t)clamp255((L + cr * E) >> 16);   // >> of a negative int: arithmetic (floor)
    rgb[1] = (uint8_t)clamp255((L - gu * D - gv * E) >> 16);
    rgb[2] = (uint8_t)clamp255((L + bu * D) >> 16);
  }
#endif
};

// The reader of one sample type: what the templated consumers (stem loader, ingest, conversion)
// read pixels through.
template <typename T>
struct YuvReader {
  YuvLayout l;
#ifdef __CUDACC__
  __device__ __forceinline__ void pixel(long long f, int r, int c, uint8_t (&rgb)[3]) const {
    l.pixel<T>(f, r, c, rgb);
  }
#endif
};

// Validates the descriptor for `frames` frames (1 + message on bad input); nothing is launched
// unless this passed.
inline int check_yuv_frames(const tapir_yuv_frames* s, int frames, const char* who) {
  TAPIR_CHECK_ARG(s != nullptr && s->y != nullptr && s->u != nullptr && s->v != nullptr,
                  "%s: null pointer", who);
  TAPIR_CHECK_ARG(frames > 0, "%s: frames=%d", who, frames);
  TAPIR_CHECK_ARG(s->H > 0 && s->W > 0 && s->h > 0 && s->w > 0,
                  "%s: zero or negative size (frame %dx%d, window %dx%d)", who, s->H, s->W, s->h, s->w);
  TAPIR_CHECK_ARG(s->y0 >= 0 && s->x0 >= 0 && (long long)s->y0 + s->h <= s->H &&
                      (long long)s->x0 + s->w <= s->W,
                  "%s: crop (%d,%d,%d,%d) outside the %dx%d frame", who, s->y0, s->x0, s->h, s->w,
                  s->H, s->W);
  TAPIR_CHECK_ARG(s->sample_bytes == 1 || s->sample_bytes == 2, "%s: sample_bytes must be 1 or 2, got %d",
                  who, s->sample_bytes);
  TAPIR_CHECK_ARG(s->bits >= 8 && s->bits <= 16 && (s->sample_bytes == 2 || s->bits == 8),
                  "%s: bits=%d with %d-byte samples (8 for 1 byte, 8..16 for 2)", who, s->bits,
                  s->sample_bytes);
  TAPIR_CHECK_ARG(s->lsb_aligned == 0 || s->lsb_aligned == 1, "%s: lsb_aligned must be 0 or 1", who);
  TAPIR_CHECK_ARG((s->chroma_shift_x == 0 || s->chroma_shift_x == 1) &&
                      (s->chroma_shift_y == 0 || s->chroma_shift_y == 1),
                  "%s: chroma shifts must be 0 or 1, got (%d, %d)", who, s->chroma_shift_x,
                  s->chroma_shift_y);
  TAPIR_CHECK_ARG(s->luma_step >= 1 && s->chroma_step >= 1, "%s: luma_step %d, chroma_step %d (>= 1)",
                  who, s->luma_step, s->chroma_step);
  TAPIR_CHECK_ARG(s->luma_step != 2 || (s->W % 2 == 0 && s->x0 % 2 == 0 && s->w % 2 == 0),
                  "%s: packed 4:2:2 rows (luma_step 2) need an even width and window column / width "
                  "(frame W=%d, window x0=%d w=%d)", who, s->W, s->x0, s->w);
  TAPIR_CHECK_ARG(s->matrix == 601 || s->matrix == 709 || s->matrix == 2020,
                  "%s: matrix must be 601, 709 or 2020, got %d", who, s->matrix);
  TAPIR_CHECK_ARG(s->full_range == 0 || s->full_range == 1, "%s: full_range must be 0 or 1", who);
  const long long b = s->sample_bytes;
  const long long cw = (s->W + (1 << s->chroma_shift_x) - 1) >> s->chroma_shift_x;
  TAPIR_CHECK_ARG(s->y_pitch >= ((s->W - 1) * (long long)s->luma_step + 1) * b &&
                      s->u_pitch >= ((cw - 1) * s->chroma_step + 1) * b &&
                      s->v_pitch >= ((cw - 1) * s->chroma_step + 1) * b,
                  "%s: row pitch smaller than a row (y %lld, u %lld, v %lld bytes for W=%d)", who,
                  (long long)s->y_pitch, (long long)s->u_pitch, (long long)s->v_pitch, s->W);
  TAPIR_CHECK_ARG(s->y_frame_stride >= 0 && s->u_frame_stride >= 0 && s->v_frame_stride >= 0,
                  "%s: negative frame stride", who);
  if (b == 2) {
    const unsigned long long any = reinterpret_cast<uintptr_t>(s->y) | reinterpret_cast<uintptr_t>(s->u) |
                                   reinterpret_cast<uintptr_t>(s->v) | s->y_pitch | s->u_pitch |
                                   s->v_pitch | s->y_frame_stride | s->u_frame_stride |
                                   s->v_frame_stride;
    TAPIR_CHECK_ARG((any & 1) == 0, "%s: 16-bit planes, pitches and frame strides must be 2-byte "
                    "aligned", who);
  }
  return kOk;
}

// The device form of a descriptor check_yuv_frames accepted.
inline YuvLayout yuv_layout(const tapir_yuv_frames& s) {
  static const int kCoef[3][2][4] = {{{409, 100, 208, 516}, {359, 88, 183, 454}},   // BT.601
                                     {{459, 55, 136, 541}, {403, 48, 120, 475}},    // BT.709
                                     {{430, 48, 167, 548}, {377, 42, 146, 482}}};   // BT.2020
  const int* c = kCoef[s.matrix == 601 ? 0 : (s.matrix == 709 ? 1 : 2)][s.full_range];
  const long long b = s.sample_bytes;
  const bool lsb = b == 2 && s.lsb_aligned;
  return YuvLayout{s.y, s.u, s.v,
                   s.y_frame_stride / b, s.u_frame_stride / b, s.v_frame_stride / b,
                   s.y_pitch / b, s.u_pitch / b, s.v_pitch / b,
                   s.luma_step, s.chroma_step, s.chroma_shift_x, s.chroma_shift_y, s.y0, s.x0,
                   b == 1 ? 0xff : (lsb ? (1 << s.bits) - 1 : 0xffff),
                   b == 1 ? 8 : (lsb ? 16 - s.bits : 0),
                   s.full_range ? 256 : 298, s.full_range ? 0 : 4096,
                   c[0], c[1], c[2], c[3]};
}

// Bytes of one frame's crop window, all three planes (for the profiler's byte counts).
inline double yuv_window_bytes(const tapir_yuv_frames& s) {
  return (double)s.h * s.w * s.sample_bytes * (1.0 + 2.0 / (1 << (s.chroma_shift_x + s.chroma_shift_y)));
}

// The tapir_yuv_frames of an 8-bit 4:2:0 descriptor (1 + message if it is no valid one): the
// 4:2:0 entry points run the general path on it.
inline int yuv_from_yuv420(const tapir_yuv420_frames* s, const char* who, tapir_yuv_frames* out) {
  TAPIR_CHECK_ARG(s != nullptr, "%s: null pointer", who);
  TAPIR_CHECK_ARG(s->chroma_step == 1 || s->chroma_step == 2,
                  "%s: chroma_step must be 1 (I420) or 2 (NV12), got %d", who, s->chroma_step);
  TAPIR_CHECK_ARG(s->matrix == 601 || s->matrix == 709, "%s: matrix must be 601 or 709, got %d",
                  who, s->matrix);
  *out = tapir_yuv_frames{s->y, s->u, s->v,
                          s->y_frame_stride, s->u_frame_stride, s->v_frame_stride,
                          s->y_pitch, s->u_pitch, s->v_pitch,
                          s->H, s->W, s->y0, s->x0, s->h, s->w, s->matrix, s->full_range,
                          /*sample_bytes=*/1, /*bits=*/8, /*lsb_aligned=*/0, /*luma_step=*/1,
                          s->chroma_step, /*chroma_shift_x=*/1, /*chroma_shift_y=*/1, 0};
  return kOk;
}

}  // namespace tapir
