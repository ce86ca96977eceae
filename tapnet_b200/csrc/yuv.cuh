// 8-bit YUV 4:2:0 -> uint8 RGB (the contract of tapir_yuv420_frames in include/tapir_b200.h),
// shared by the stem conv's loader (backbone.cu) and the ingest / conversion kernels
// (frames_io.cu).  Integer arithmetic only, so every reader produces the same bytes.
#pragma once
#include "../../include/tapir_b200.h"
#include "common.cuh"

namespace tapir {

// A crop window of tapir_yuv420_frames as the kernels read it: pixel(f, r, c) is window pixel
// (r, c) of frame f, i.e. frame pixel (y0 + r, x0 + c).
struct Yuv420Reader {
  const uint8_t* y;
  const uint8_t* u;
  const uint8_t* v;
  long long y_frame, u_frame, v_frame;
  long long y_pitch, u_pitch, v_pitch;
  int step, y0, x0;
  int k, c_off;          // luma gain and offset: (298, 16) limited range, (256, 0) full range
  int cr, gu, gv, bu;    // chroma coefficients (R from V, G from U and V, B from U)

#ifdef __CUDACC__
  __device__ __forceinline__ static int clamp255(int x) { return x < 0 ? 0 : (x > 255 ? 255 : x); }

  __device__ __forceinline__ void pixel(long long f, int r, int c, uint8_t (&rgb)[3]) const {
    const int ay = y0 + r, ax = x0 + c;
    const long long cy = ay >> 1, cx = (long long)(ax >> 1) * step;
    const int Y = __ldg(y + f * y_frame + ay * y_pitch + ax);
    const int D = (int)__ldg(u + f * u_frame + cy * u_pitch + cx) - 128;
    const int E = (int)__ldg(v + f * v_frame + cy * v_pitch + cx) - 128;
    const int L = k * (Y - c_off) + 128;
    rgb[0] = (uint8_t)clamp255((L + cr * E) >> 8);   // >> of a negative int: arithmetic (floor)
    rgb[1] = (uint8_t)clamp255((L - gu * D - gv * E) >> 8);
    rgb[2] = (uint8_t)clamp255((L + bu * D) >> 8);
  }
#endif
};

// Validates the descriptor (1 + message on bad input) and fills the reader.
inline int make_yuv420_reader(const tapir_yuv420_frames* s, int frames, const char* who,
                              Yuv420Reader* r) {
  TAPIR_CHECK_ARG(s != nullptr && s->y != nullptr && s->u != nullptr && s->v != nullptr,
                  "%s: null pointer", who);
  TAPIR_CHECK_ARG(frames > 0, "%s: frames=%d", who, frames);
  TAPIR_CHECK_ARG(s->H > 0 && s->W > 0 && s->h > 0 && s->w > 0,
                  "%s: zero or negative size (frame %dx%d, window %dx%d)", who, s->H, s->W, s->h, s->w);
  TAPIR_CHECK_ARG(s->y0 >= 0 && s->x0 >= 0 && (long long)s->y0 + s->h <= s->H &&
                      (long long)s->x0 + s->w <= s->W,
                  "%s: crop (%d,%d,%d,%d) outside the %dx%d frame", who, s->y0, s->x0, s->h, s->w,
                  s->H, s->W);
  TAPIR_CHECK_ARG(s->chroma_step == 1 || s->chroma_step == 2,
                  "%s: chroma_step must be 1 (I420) or 2 (NV12), got %d", who, s->chroma_step);
  TAPIR_CHECK_ARG(s->matrix == 601 || s->matrix == 709, "%s: matrix must be 601 or 709, got %d",
                  who, s->matrix);
  TAPIR_CHECK_ARG(s->full_range == 0 || s->full_range == 1, "%s: full_range must be 0 or 1", who);
  const long long cw = (s->W + 1) / 2;
  TAPIR_CHECK_ARG(s->y_pitch >= s->W && s->u_pitch >= (cw - 1) * s->chroma_step + 1 &&
                      s->v_pitch >= (cw - 1) * s->chroma_step + 1,
                  "%s: row pitch smaller than a row (y %lld, u %lld, v %lld for W=%d)", who,
                  (long long)s->y_pitch, (long long)s->u_pitch, (long long)s->v_pitch, s->W);
  TAPIR_CHECK_ARG(s->y_frame_stride >= 0 && s->u_frame_stride >= 0 && s->v_frame_stride >= 0,
                  "%s: negative frame stride", who);
  static const int kCoef[2][2][4] = {{{409, 100, 208, 516}, {359, 88, 183, 454}},   // BT.601
                                     {{459, 55, 136, 541}, {403, 48, 120, 475}}};   // BT.709
  const int* c = kCoef[s->matrix == 709][s->full_range];
  *r = Yuv420Reader{s->y, s->u, s->v,
                    s->y_frame_stride, s->u_frame_stride, s->v_frame_stride,
                    s->y_pitch, s->u_pitch, s->v_pitch,
                    s->chroma_step, s->y0, s->x0,
                    s->full_range ? 256 : 298, s->full_range ? 0 : 16,
                    c[0], c[1], c[2], c[3]};
  return kOk;
}

}  // namespace tapir
