// Internal C++ interface of the hot-path kernels (everything here is reached only through
// the extern "C" functions of api.cu / include/tapir_b200.h).
#pragma once
#include "../../include/tapir_b200.h"
#include "common.cuh"
#include "gemm.cuh"
#include "yuv.cuh"

namespace tapir {

// Bump allocator over caller-provided workspace; with base == nullptr it only measures.
struct Arena {
  char* base;
  size_t off;
  size_t cap;
  bool ok;
  Arena(void* b, size_t c) : base(static_cast<char*>(b)), off(0), cap(c), ok(true) {}
  template <typename T>
  T* take(size_t n) {
    off = align_up(off, 256);
    T* p = base ? reinterpret_cast<T*>(base + off) : nullptr;
    off += n * sizeof(T);
    if (base && off > cap) ok = false;
    return p;
  }
};

// ---- elementwise / normalisation (backbone.cu) ------------------------------------------
int split_planes(const float* src, long long ld_src, __nv_bfloat16* dst, long long ld_dst,
                 long long plane_stride, long long rows, int cols, int cols_padded, int planes,
                 cudaStream_t s);
int stem_conv(const void* video, int video_u8, const float* w_packed, int frames, int H, int W,
              float* out, cudaStream_t s);
// the stem conv on the H x W crop window of YUV frames (converted inside the patch loads); the
// descriptor passed check_yuv_frames
int stem_conv_yuv(const tapir_yuv_frames& video, const float* w_packed, int frames, int H, int W,
                  float* out, cudaStream_t s);
int instnorm_stats(const float* x, int frames, long long hw, int C, double* sums, cudaStream_t s);
int instnorm_relu_split(const float* x, const double* sums, const float* w, const float* b,
                        int frames, long long hw, int C, __nv_bfloat16* out, long long plane_stride,
                        int planes, double* zero_next, int zero_channels, cudaStream_t s);
int im2col_s2(const __nv_bfloat16* in, long long in_plane_stride, int frames, int H, int W, int C,
              int taps, __nv_bfloat16* out, long long out_plane_stride, int planes, cudaStream_t s);
int layernorm_split(const float* x, long long rows, int C, const float* w, const float* b,
                    float* y, __nv_bfloat16* planes_out, long long plane_stride, int planes,
                    cudaStream_t s);
int l2_normalize(const float* x, long long rows, int C, float* out, cudaStream_t s);
int bilinear_resize(const float* src, int frames, int H, int W, int C, float* dst, int oH, int oW,
                    cudaStream_t s);
size_t backbone_workspace_bytes(int frames, int H, int W, int extra_convs, int planes);
int backbone_stem(const tapir_backbone_weights* w, const void* video_chunk, int video_u8,
                  int pass_frames, int H, int W, int frame0, int nframes, void* ws, size_t ws_bytes,
                  cudaStream_t s);
int backbone_forward(const tapir_backbone_weights* w, const void* video, int video_u8, int frames,
                     int H, int W, float* lowres, float* hires, void* ws, size_t ws_bytes,
                     cudaStream_t s, cudaEvent_t hires_ready = nullptr,
                     const tapir_yuv_frames* yuv = nullptr);

// ---- callers either side of the path (frames_io.cu; SURVEY 8f rows 1, 2) ----------------
int ingest_frames(const uint8_t* src, int frames, int H, int W, int crop_y, int crop_x, int crop_h,
                  int crop_w, float* dst, int oH, int oW, cudaStream_t s);
// YUV descriptors that passed check_yuv_frames
int ingest_frames_yuv(const tapir_yuv_frames& src, int frames, float* dst, int oH, int oW,
                      cudaStream_t s);
int yuv_to_rgb(const tapir_yuv_frames& src, int frames, uint8_t* dst, cudaStream_t s);
int ingest_frames_multi(const tapir_ingest_desc* descs, int frames, float* dst, int oH, int oW,
                        cudaStream_t s);
int postprocess_occlusions(const float* occ, const float* expd, long long n, uint8_t* visible,
                           cudaStream_t s);
int tapvid_counts(const tapir_tapvid_args* a, cudaStream_t s);
int redetection_max_events(int T);
int redetection_events(const tapir_redetection_args* a, cudaStream_t s);

// ---- camera homographies from point tracks (homography.cu; viz_utils.py:301-648) -----------
size_t homographies_workspace_bytes(int T, int N);
// Host only: the RANSAC stop table thr[it] = min(1 - (it + 1) / N, frac * pow(0.99, it)) * N.
void ransac_stop_thresholds(int N, double frac, double* out);
// Arguments checked by tapir_homographies_wrt_frame.
int homographies_wrt_frame(const tapir_homography_args* a, cudaStream_t s);

// ---- Lanczos resize of uint8 RGB clips (resample.cu; PIL's 8-bit LANCZOS) -------------------
// Host only: the per-axis kernel width, and the (xmin, n) bounds [out][2] and 22-bit fixed-point
// taps [out][ksize] of one axis.
int lanczos_ksize(int in_size, int out_size);
void lanczos_weights(int in_size, int out_size, int* bounds, int* taps);
size_t resize_lanczos_u8_workspace_bytes(int frames, int H, int W, int h, int w);
// Arguments checked by tapir_resize_lanczos_u8.
int resize_lanczos_u8(const uint8_t* src, uint8_t* dst, int frames, int H, int W, int h, int w,
                      const int* x_bounds, const int* x_taps, int x_ksize, const int* y_bounds,
                      const int* y_taps, int y_ksize, uint8_t* ws, cudaStream_t s);

// ---- point-track painting (paint.cu; viz_utils.py:47-124) ---------------------------------
int paint_radius(int H, int W);
size_t paint_point_track_workspace_bytes(long long frames, long long points);
// Arguments checked by tapir_paint_point_track; T * ceil(H/32) * ceil(W/32) fits a grid.
int paint_point_track(const uint8_t* frames, int T, int H, int W, const void* tracks, int tracks_fp64,
                      const uint8_t* visibles, int N, const uint8_t* colors, uint8_t* out, void* ws,
                      cudaStream_t s);

// ---- stage A (stage_a.cu) ---------------------------------------------------------------
// frame_slot: null (the grid holds all T frames of the clip) or vT entries, each frame's slot
// among the grid's T or -1 (see sample_query_kernel)
int sample_query_features(const float* grid, int T, int gh, int gw, int C, const float* query_tyx,
                          int N, int vT, int vH, int vW, const int* frame_slot, float* out,
                          cudaStream_t s);
// Arguments checked by tapir_sample_query_rows: num_grids in 1..TAPIR_MAX_QUERY_GRIDS, state a
// device table of num_state (even) row-aligned tensors.
int sample_query_rows(const tapir_query_grid* grids, int num_grids, int clips, int rows, int video_h,
                      int video_w, const int32_t* video_hw, const int32_t* count,
                      const tapir_query_request* requests, float* const* state, int num_state,
                      cudaStream_t s);
// B clips: qfeat [B][N][C], grid [B][T][gh][gw][C], outputs indexed by flattened query b*N + n
// (the workspace of B clips with Q queries in all)
size_t cost_volume_workspace_bytes(int B, long long Q, int T, int gh, int gw, int C);
int cost_volume_tracks(const tapir_head_weights* w, const float* qfeat, const float* grid, int B,
                       int N, int T, int gh, int gw, int C, const float* query_tyx, float temperature,
                       int init_h, int init_w, float* points, float* occ, float* expd, int* argmax,
                       void* ws, size_t ws_bytes, cudaStream_t s);
// B <= kGemmMaxGroups clips of counts[b] (host) queries each, one after the other in qfeat [Q][C]
int cost_volume_tracks_ragged(const tapir_head_weights* w, const float* qfeat, const float* grid, int B,
                              const int* counts, int T, int gh, int gw, int C, const float* query_tyx,
                              float temperature, int init_h, int init_w, float* points, float* occ,
                              float* expd, int* argmax, void* ws, size_t ws_bytes, cudaStream_t s);

// ---- refinement (refine.cu) -------------------------------------------------------------
int pool_pyramid(const float* grid, int T, int h, int w, int C, float* out, cudaStream_t s);
// a->num_points queries per clip, `batch` clips; level grids are [batch][T][h][w][C].  With a
// device table query_clip [a->num_points], a->num_points is the queries of all clips and query q
// reads the grids of clip query_clip[q].
int local_corr(const tapir_corr_args* a, int batch, cudaStream_t s, const int32_t* query_clip = nullptr);
size_t mixer_workspace_bytes(long long rows, int planes);
int mixer_forward(const tapir_mixer_weights* w, const tapir_mixer_io* io, void* ws, size_t ws_bytes,
                  cudaStream_t s);
// The depthwise half of one mixer block (everything before its channel MLP) on x [n][T][512]:
// z [n][T][512] and LN_1(z) * w as bf16 planes [planes][n*T][512].  Context pointers: causal only.
int mixer_dw(const tapir_mixer_block& blk, const float* x, int n, int T, bool causal, const float* ctx1_in,
             const float* ctx2_in, float* ctx1_out, float* ctx2_out, float* z, __nv_bfloat16* planes_out,
             long long plane_stride, int planes, cudaStream_t s);
// video_hw: NULL, or a device table [clips][2] of per-clip video sizes (rows_per_clip rows each,
// or, with a device table query_clip [a->num_points], query q's rows are clip query_clip[q]'s)
int refine_update(const tapir_update_args* a, cudaStream_t s, const int32_t* video_hw = nullptr,
                  long long rows_per_clip = 0, const int32_t* query_clip = nullptr);

}  // namespace tapir
