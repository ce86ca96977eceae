// extern "C" surface of libtapir_b200.so (include/tapir_b200.h).
#include <nvtx3/nvToolsExt.h>

#include <cmath>

#include "kernels.cuh"

namespace tapir {
const char* last_error();
void profile_enable(int on);
int profile_report(char* buf, size_t cap);
}

using namespace tapir;

namespace {
inline cudaStream_t S(void* s) { return static_cast<cudaStream_t>(s); }

// NVTX range per stage (SURVEY.md section 5): shows up in nsys / ncu --nvtx timelines, costs one
// predictable branch when no tool is attached (header-only NVTX v3, injection library loaded lazily).
struct Range {
  explicit Range(const char* name) { nvtxRangePushA(name); }
  ~Range() { nvtxRangePop(); }
};
}  // namespace

extern "C" {

const char* tapir_last_error(void) { return tapir::last_error(); }
int tapir_abi_version(void) { return TAPIR_B200_ABI_VERSION; }
unsigned long long tapir_launch_count(void) { return tapir::g_launch_count; }

void tapir_profile_enable(int32_t on) { tapir::profile_enable(on); }
int tapir_profile_report(char* buf, size_t capacity) { return tapir::profile_report(buf, capacity); }

int tapir_split_planes(const float* src, int64_t ld_src, void* dst, int64_t ld_dst,
                       int64_t plane_stride, int64_t rows, int32_t cols, int32_t cols_padded,
                       int32_t planes, void* stream) {
  Range nvtx_range("tapir_split_planes");
  TAPIR_CHECK_ARG(src != nullptr && dst != nullptr, "tapir_split_planes: null pointer");
  return split_planes(src, ld_src, static_cast<__nv_bfloat16*>(dst), ld_dst, plane_stride, rows, cols,
                      cols_padded, planes, S(stream));
}

int tapir_gemm(const void* a_planes, int32_t lda, int64_t a_plane_stride, const tapir_linear* b,
               int64_t M, int32_t conv3x3, int32_t frames, int32_t H, int32_t W, int32_t C,
               const float* residual, int32_t ldr, int32_t act_gelu, float* out_f32, int32_t ldo,
               void* out_planes, int32_t ldp, int64_t out_plane_stride, int32_t out_P,
               double* stats, int32_t rows_per_frame, int32_t impl, void* stream) {
  return tapir_gemm_ex(a_planes, lda, a_plane_stride, b, M, conv3x3, frames, H, W, C, residual, ldr,
                       act_gelu, out_f32, ldo, out_planes, ldp, out_plane_stride, out_P, stats,
                       rows_per_frame, impl, nullptr, 0, stream);
}

int tapir_gemm_ex(const void* a_planes, int32_t lda, int64_t a_plane_stride, const tapir_linear* b,
                  int64_t M, int32_t conv3x3, int32_t frames, int32_t H, int32_t W, int32_t C,
                  const float* residual, int32_t ldr, int32_t act_gelu, float* out_f32,
                  int32_t ldo, void* out_planes, int32_t ldp, int64_t out_plane_stride,
                  int32_t out_P, double* stats, int32_t rows_per_frame, int32_t impl,
                  void* splitk_workspace, size_t splitk_workspace_bytes, void* stream) {
  Range nvtx_range("tapir_gemm");
  TAPIR_CHECK_ARG(a_planes != nullptr && b != nullptr && b->w != nullptr, "tapir_gemm: null pointer");
  TAPIR_CHECK_ARG(M > 0 && M < (1ll << 31), "tapir_gemm: M out of range");
  TAPIR_CHECK_ARG((reinterpret_cast<uintptr_t>(splitk_workspace) & 15) == 0,
                  "tapir_gemm: split-K workspace must be 16-byte aligned");
  GemmArgs g = gemm_args(*b);
  g.mode = conv3x3 ? kGemmConv3x3 : kGemmPlain;
  g.M = (int)M;
  g.a = static_cast<const __nv_bfloat16*>(a_planes);
  g.lda = lda;
  g.a_plane_stride = a_plane_stride;
  g.frames = frames; g.H = H; g.W = W; g.C = C;
  g.residual = residual; g.ldr = ldr;
  g.act = act_gelu ? 1 : 0;
  g.out_f32 = out_f32; g.ldo = ldo;
  g.out_planes = static_cast<__nv_bfloat16*>(out_planes);
  g.ldp = ldp; g.out_plane_stride = out_plane_stride; g.out_P = out_P;
  g.stats = stats; g.rows_per_frame = rows_per_frame;
  g.splitk_ws = static_cast<float*>(splitk_workspace);
  g.splitk_ws_bytes = splitk_workspace != nullptr ? splitk_workspace_bytes : 0;
  g.allow_splitk = splitk_workspace != nullptr;
  GemmSwitches sw;  // validated here whichever kernel `impl` names; sw.simt is not used
  TAPIR_RETURN_IF(read_gemm_switches(&sw));
  if (impl == 1) return gemm_simt(g, S(stream));
  if (impl == 0) return gemm_tc(g, sw, S(stream));
  set_error("tapir_gemm: impl must be 0 (wgmma) or 1 (simt)");
  return kBadArgument;
}

int tapir_bilinear_resize(const float* src, int32_t frames, int32_t H, int32_t W, int32_t C,
                          float* dst, int32_t oH, int32_t oW, void* stream) {
  Range nvtx_range("tapir_bilinear_resize");
  TAPIR_CHECK_ARG(src && dst && frames > 0 && H > 0 && W > 0 && C > 0 && oH > 0 && oW > 0,
                  "tapir_bilinear_resize: bad arguments");
  return bilinear_resize(src, frames, H, W, C, dst, oH, oW, S(stream));
}

// The backbone's HBM-bound building blocks.  The internal functions trust their callers
// (backbone_forward, mixer_forward); these entry points check every argument first, so a bad one
// returns kBadArgument before any CUDA call.
namespace {
constexpr int kMaxGridFrames = 65535;  // frames run on gridDim.y / gridDim.z

bool aligned(const void* p, int bytes) { return (reinterpret_cast<uintptr_t>(p) % bytes) == 0; }
bool overlap(const void* a, size_t a_bytes, const void* b, size_t b_bytes) {
  const uintptr_t pa = reinterpret_cast<uintptr_t>(a), pb = reinterpret_cast<uintptr_t>(b);
  return pa < pb + b_bytes && pb < pa + a_bytes;
}
}  // namespace

int tapir_stem_conv(const void* video, int32_t video_u8, const float* w_packed, int32_t frames,
                    int32_t H, int32_t W, float* out, void* stream) {
  Range nvtx_range("tapir_stem_conv");
  TAPIR_CHECK_ARG(video && w_packed && out, "tapir_stem_conv: null pointer");
  TAPIR_CHECK_ARG(frames > 0 && frames <= kMaxGridFrames, "tapir_stem_conv: frames=%d", frames);
  TAPIR_CHECK_ARG(H > 0 && W > 0 && H % 2 == 0 && W % 2 == 0,
                  "tapir_stem_conv: H=%d W=%d must be positive and even", H, W);
  TAPIR_CHECK_ARG(aligned(out, 16) && (video_u8 || aligned(video, 4)),
                  "tapir_stem_conv: out must be 16-byte aligned, a float video 4-byte aligned");
  return stem_conv(video, video_u8 ? 1 : 0, w_packed, frames, H, W, out, S(stream));
}

int tapir_instnorm_stats(const float* x, int32_t frames, int64_t hw, int32_t C, double* sums,
                         void* stream) {
  Range nvtx_range("tapir_instnorm_stats");
  TAPIR_CHECK_ARG(x && sums, "tapir_instnorm_stats: null pointer");
  TAPIR_CHECK_ARG(frames > 0 && frames <= kMaxGridFrames && hw > 0,
                  "tapir_instnorm_stats: frames=%d hw=%lld", frames, (long long)hw);
  TAPIR_CHECK_ARG(C == 64 || C == 128 || C == 256, "tapir_instnorm_stats: C=%d unsupported", C);
  TAPIR_CHECK_ARG(aligned(x, 16) && aligned(sums, 8),
                  "tapir_instnorm_stats: x must be 16-byte and sums 8-byte aligned");
  return instnorm_stats(x, frames, hw, C, sums, S(stream));
}

int tapir_instnorm_relu_split(const float* x, const double* sums, const float* w, const float* b,
                              int32_t frames, int64_t hw, int32_t C, void* out_planes,
                              int64_t plane_stride, int32_t planes, double* zero_next,
                              int32_t zero_channels, void* stream) {
  Range nvtx_range("tapir_instnorm_relu_split");
  TAPIR_CHECK_ARG(x && sums && w && b && out_planes, "tapir_instnorm_relu_split: null pointer");
  TAPIR_CHECK_ARG(frames > 0 && frames <= kMaxGridFrames && hw > 0,
                  "tapir_instnorm_relu_split: frames=%d hw=%lld", frames, (long long)hw);
  TAPIR_CHECK_ARG(C == 64 || C == 128 || C == 256, "tapir_instnorm_relu_split: C=%d unsupported", C);
  TAPIR_CHECK_ARG(planes >= 1 && planes <= 3, "tapir_instnorm_relu_split: planes=%d", planes);
  TAPIR_CHECK_ARG(planes == 1 || plane_stride >= (long long)frames * hw * C,
                  "tapir_instnorm_relu_split: planes overlap (plane_stride=%lld)", (long long)plane_stride);
  TAPIR_CHECK_ARG(aligned(x, 16) && aligned(sums, 8) && aligned(out_planes, 8) && plane_stride % 4 == 0,
                  "tapir_instnorm_relu_split: x must be 16-byte aligned, sums and out_planes 8-byte "
                  "aligned, plane_stride a multiple of 4");
  TAPIR_CHECK_ARG(zero_next == nullptr || (zero_channels > 0 && aligned(zero_next, 8)),
                  "tapir_instnorm_relu_split: zero_next needs zero_channels > 0 and 8-byte alignment");
  return instnorm_relu_split(x, sums, w, b, frames, hw, C, static_cast<__nv_bfloat16*>(out_planes),
                             plane_stride, planes, zero_next, zero_channels, S(stream));
}

int tapir_im2col_s2(const void* in_planes, int64_t in_plane_stride, int32_t frames, int32_t H,
                    int32_t W, int32_t C, int32_t taps, void* out_planes, int64_t out_plane_stride,
                    int32_t planes, void* stream) {
  Range nvtx_range("tapir_im2col_s2");
  TAPIR_CHECK_ARG(in_planes && out_planes, "tapir_im2col_s2: null pointer");
  TAPIR_CHECK_ARG(frames > 0 && H > 0 && W > 0 && H % 2 == 0 && W % 2 == 0,
                  "tapir_im2col_s2: frames=%d H=%d W=%d (H, W positive and even)", frames, H, W);
  TAPIR_CHECK_ARG(C > 0 && C % 8 == 0, "tapir_im2col_s2: C=%d must be a positive multiple of 8", C);
  TAPIR_CHECK_ARG(taps == 1 || taps == 9, "tapir_im2col_s2: taps=%d must be 1 or 9", taps);
  TAPIR_CHECK_ARG(planes >= 1 && planes <= 3, "tapir_im2col_s2: planes=%d", planes);
  TAPIR_CHECK_ARG(aligned(in_planes, 16) && aligned(out_planes, 16) && in_plane_stride % 8 == 0 &&
                      out_plane_stride % 8 == 0,
                  "tapir_im2col_s2: planes must be 16-byte aligned, plane strides multiples of 8");
  return im2col_s2(static_cast<const __nv_bfloat16*>(in_planes), in_plane_stride, frames, H, W, C, taps,
                   static_cast<__nv_bfloat16*>(out_planes), out_plane_stride, planes, S(stream));
}

int tapir_layernorm_split(const float* x, int64_t rows, int32_t C, const float* w, const float* b,
                          float* y, void* planes_out, int64_t plane_stride, int32_t planes,
                          void* stream) {
  Range nvtx_range("tapir_layernorm_split");
  TAPIR_CHECK_ARG(x && w, "tapir_layernorm_split: null pointer");
  TAPIR_CHECK_ARG(y || planes_out, "tapir_layernorm_split: y and planes_out are both NULL");
  TAPIR_CHECK_ARG(rows > 0 && rows < (1ll << 34), "tapir_layernorm_split: rows=%lld", (long long)rows);
  TAPIR_CHECK_ARG(C == 256 || C == 512, "tapir_layernorm_split: C=%d unsupported", C);
  TAPIR_CHECK_ARG(planes_out == nullptr || (planes >= 1 && planes <= 3),
                  "tapir_layernorm_split: planes=%d", planes);
  TAPIR_CHECK_ARG(planes_out == nullptr || planes == 1 || plane_stride >= rows * C,
                  "tapir_layernorm_split: planes overlap (plane_stride=%lld)", (long long)plane_stride);
  TAPIR_CHECK_ARG(aligned(x, 16) && aligned(w, 16) && aligned(b, 16) && aligned(y, 16) &&
                      aligned(planes_out, 8) && plane_stride % 4 == 0,
                  "tapir_layernorm_split: x, w, b, y must be 16-byte aligned, planes_out 8-byte "
                  "aligned, plane_stride a multiple of 4");
  return layernorm_split(x, rows, C, w, b, y, static_cast<__nv_bfloat16*>(planes_out), plane_stride,
                         planes_out ? planes : 0, S(stream));
}

int tapir_l2_normalize(const float* x, int64_t rows, int32_t C, float* out, void* stream) {
  Range nvtx_range("tapir_l2_normalize");
  TAPIR_CHECK_ARG(x && out, "tapir_l2_normalize: null pointer");
  TAPIR_CHECK_ARG(rows > 0 && rows < (1ll << 34), "tapir_l2_normalize: rows=%lld", (long long)rows);
  TAPIR_CHECK_ARG(C == 128 || C == 256, "tapir_l2_normalize: C=%d unsupported", C);
  TAPIR_CHECK_ARG(aligned(x, 16) && aligned(out, 16), "tapir_l2_normalize: x and out must be 16-byte aligned");
  return l2_normalize(x, rows, C, out, S(stream));
}

size_t tapir_backbone_workspace_bytes(int32_t frames, int32_t H, int32_t W, int32_t extra_convs,
                                      int32_t planes) {
  return backbone_workspace_bytes(frames, H, W, extra_convs, planes);
}

int tapir_backbone_forward(const tapir_backbone_weights* w, const float* video, int32_t frames,
                           int32_t H, int32_t W, float* lowres, float* hires, void* workspace,
                           size_t workspace_bytes, void* stream) {
  Range nvtx_range("tapir_backbone_forward");
  return backbone_forward(w, video, 0, frames, H, W, lowres, hires, workspace, workspace_bytes, S(stream));
}

int tapir_backbone_forward_u8(const tapir_backbone_weights* w, const uint8_t* video,
                              int32_t frames, int32_t H, int32_t W, float* lowres, float* hires,
                              void* workspace, size_t workspace_bytes, void* stream) {
  Range nvtx_range("tapir_backbone_forward_u8");
  return backbone_forward(w, video, 1, frames, H, W, lowres, hires, workspace, workspace_bytes, S(stream));
}

int tapir_backbone_forward_ex(const tapir_backbone_weights* w, const void* video, int32_t video_u8,
                              int32_t frames, int32_t H, int32_t W, float* lowres, float* hires,
                              void* workspace, size_t workspace_bytes, void* hires_ready_event,
                              void* stream) {
  Range nvtx_range("tapir_backbone_forward_ex");
  return backbone_forward(w, video, video_u8 ? 1 : 0, frames, H, W, lowres, hires, workspace,
                          workspace_bytes, S(stream), static_cast<cudaEvent_t>(hires_ready_event));
}

int tapir_backbone_stem(const tapir_backbone_weights* w, const void* video_chunk, int32_t video_u8,
                        int32_t pass_frames, int32_t H, int32_t W, int32_t frame0, int32_t nframes,
                        void* workspace, size_t workspace_bytes, void* stream) {
  Range nvtx_range("tapir_backbone_stem");
  return backbone_stem(w, video_chunk, video_u8 ? 1 : 0, pass_frames, H, W, frame0, nframes, workspace,
                       workspace_bytes, S(stream));
}

int tapir_ingest_frames(const uint8_t* src, int32_t frames, int32_t H, int32_t W, int32_t crop_y,
                        int32_t crop_x, int32_t crop_h, int32_t crop_w, float* dst, int32_t oH,
                        int32_t oW, void* stream) {
  Range nvtx_range("tapir_ingest_frames");
  return ingest_frames(src, frames, H, W, crop_y, crop_x, crop_h, crop_w, dst, oH, oW, S(stream));
}

int tapir_yuv_to_rgb(const tapir_yuv_frames* src, int32_t frames, uint8_t* dst, void* stream) {
  Range nvtx_range("tapir_yuv_to_rgb");
  TAPIR_RETURN_IF(check_yuv_frames(src, frames, "tapir_yuv_to_rgb"));
  return yuv_to_rgb(*src, frames, dst, S(stream));
}

int tapir_yuv420_to_rgb(const tapir_yuv420_frames* src, int32_t frames, uint8_t* dst, void* stream) {
  Range nvtx_range("tapir_yuv420_to_rgb");
  tapir_yuv_frames y;
  TAPIR_RETURN_IF(yuv_from_yuv420(src, "tapir_yuv420_to_rgb", &y));
  TAPIR_RETURN_IF(check_yuv_frames(&y, frames, "tapir_yuv420_to_rgb"));
  return yuv_to_rgb(y, frames, dst, S(stream));
}

int tapir_ingest_frames_yuv(const tapir_yuv_frames* src, int32_t frames, float* dst, int32_t oH,
                            int32_t oW, void* stream) {
  Range nvtx_range("tapir_ingest_frames_yuv");
  TAPIR_RETURN_IF(check_yuv_frames(src, frames, "tapir_ingest_frames_yuv"));
  return ingest_frames_yuv(*src, frames, dst, oH, oW, S(stream));
}

int tapir_ingest_frames_yuv420(const tapir_yuv420_frames* src, int32_t frames, float* dst,
                               int32_t oH, int32_t oW, void* stream) {
  Range nvtx_range("tapir_ingest_frames_yuv420");
  tapir_yuv_frames y;
  TAPIR_RETURN_IF(yuv_from_yuv420(src, "tapir_ingest_frames_yuv420", &y));
  TAPIR_RETURN_IF(check_yuv_frames(&y, frames, "tapir_ingest_frames_yuv420"));
  return ingest_frames_yuv(y, frames, dst, oH, oW, S(stream));
}

int tapir_ingest_frames_multi(const tapir_ingest_desc* descs, int32_t frames, float* dst,
                              int32_t oH, int32_t oW, void* stream) {
  Range nvtx_range("tapir_ingest_frames_multi");
  return ingest_frames_multi(descs, frames, dst, oH, oW, S(stream));
}

int tapir_backbone_forward_yuv(const tapir_backbone_weights* w, const tapir_yuv_frames* video,
                               int32_t frames, float* lowres, float* hires, void* workspace,
                               size_t workspace_bytes, void* hires_ready_event, void* stream) {
  Range nvtx_range("tapir_backbone_forward_yuv");
  TAPIR_RETURN_IF(check_yuv_frames(video, frames, "tapir_backbone_forward_yuv"));
  return backbone_forward(w, nullptr, 0, frames, video->h, video->w, lowres, hires, workspace,
                          workspace_bytes, S(stream), static_cast<cudaEvent_t>(hires_ready_event), video);
}

int tapir_backbone_forward_yuv420(const tapir_backbone_weights* w, const tapir_yuv420_frames* video,
                                  int32_t frames, float* lowres, float* hires, void* workspace,
                                  size_t workspace_bytes, void* hires_ready_event, void* stream) {
  Range nvtx_range("tapir_backbone_forward_yuv420");
  tapir_yuv_frames y;
  TAPIR_RETURN_IF(yuv_from_yuv420(video, "tapir_backbone_forward_yuv420", &y));
  TAPIR_RETURN_IF(check_yuv_frames(&y, frames, "tapir_backbone_forward_yuv420"));
  return backbone_forward(w, nullptr, 0, frames, y.h, y.w, lowres, hires, workspace,
                          workspace_bytes, S(stream), static_cast<cudaEvent_t>(hires_ready_event), &y);
}

int tapir_postprocess_occlusions(const float* occ, const float* expd, int64_t n, uint8_t* visible,
                                 void* stream) {
  Range nvtx_range("tapir_postprocess_occlusions");
  return postprocess_occlusions(occ, expd, n, visible, S(stream));
}

int tapir_tapvid_counts(const tapir_tapvid_args* args, void* stream) {
  Range nvtx_range("tapir_tapvid_counts");
  return tapvid_counts(args, S(stream));
}

int32_t tapir_redetection_max_events(int32_t T) { return redetection_max_events(T); }

int tapir_redetection_events(const tapir_redetection_args* args, void* stream) {
  Range nvtx_range("tapir_redetection_events");
  return redetection_events(args, S(stream));
}

int tapir_sample_query_features(const float* grid, int32_t T, int32_t gh, int32_t gw, int32_t C,
                                const float* query_tyx, int32_t N, int32_t vT, int32_t vH,
                                int32_t vW, float* out, void* stream) {
  Range nvtx_range("tapir_sample_query_features");
  return sample_query_features(grid, T, gh, gw, C, query_tyx, N, vT, vH, vW, nullptr, out, S(stream));
}

int tapir_sample_query_features_ex(const float* grid, int32_t T, int32_t gh, int32_t gw, int32_t C,
                                   const float* query_tyx, int32_t N, int32_t vT, int32_t vH,
                                   int32_t vW, const int32_t* frame_slot, float* out, void* stream) {
  Range nvtx_range("tapir_sample_query_features_ex");
  const char* fn = "tapir_sample_query_features_ex";
  TAPIR_CHECK_ARG(grid && query_tyx && out, "%s: null grid, query_tyx or out", fn);
  TAPIR_CHECK_ARG(N >= 1 && T >= 1 && gh >= 1 && gw >= 1 && C >= 1,
                  "%s: N=%d T=%d gh=%d gw=%d C=%d must be positive", fn, N, T, gh, gw, C);
  TAPIR_CHECK_ARG(vT >= 1 && vH >= 1 && vW >= 1, "%s: video %d x %d x %d must be positive", fn, vT, vH, vW);
  TAPIR_CHECK_ARG(aligned(grid, 4) && aligned(query_tyx, 4) && aligned(out, 4) && aligned(frame_slot, 4),
                  "%s: grid, query_tyx, out and frame_slot must be 4-byte aligned", fn);
  const size_t out_bytes = (size_t)N * C * 4;
  TAPIR_CHECK_ARG(!overlap(out, out_bytes, grid, (size_t)T * gh * gw * C * 4) &&
                      !overlap(out, out_bytes, query_tyx, (size_t)N * 12) &&
                      !overlap(out, out_bytes, frame_slot, frame_slot ? (size_t)vT * 4 : 0),
                  "%s: out overlaps grid, query_tyx or frame_slot", fn);
  return sample_query_features(grid, T, gh, gw, C, query_tyx, N, vT, vH, vW, frame_slot, out, S(stream));
}

int tapir_sample_query_rows(const tapir_query_grid* grids, int32_t num_grids, int32_t clips,
                            int32_t rows, int32_t video_h, int32_t video_w, const int32_t* video_hw,
                            const int32_t* count, const tapir_query_request* requests,
                            float* const* state, int32_t num_state, void* stream) {
  Range nvtx_range("tapir_sample_query_rows");
  const char* fn = "tapir_sample_query_rows";
  TAPIR_CHECK_ARG(grids && num_grids >= 1 && num_grids <= TAPIR_MAX_QUERY_GRIDS,
                  "%s: %d grids, 1..%d supported", fn, num_grids, TAPIR_MAX_QUERY_GRIDS);
  TAPIR_CHECK_ARG(clips >= 1 && rows >= 1, "%s: clips=%d rows=%d must be positive", fn, clips, rows);
  TAPIR_CHECK_ARG(video_hw != nullptr || (video_h >= 1 && video_w >= 1), "%s: video %d x %d", fn, video_h,
                  video_w);
  TAPIR_CHECK_ARG(count && requests && aligned(count, 4) && aligned(requests, 4) && aligned(video_hw, 4),
                  "%s: count, requests and video_hw must be 4-byte aligned device pointers", fn);
  TAPIR_CHECK_ARG(num_state >= 0 && num_state % 2 == 0 && num_state < 65535 &&
                      (num_state == 0 || (state != nullptr && aligned(state, 8))),
                  "%s: num_state=%d must be even with an 8-byte aligned table", fn, num_state);
  for (int i = 0; i < num_grids; ++i) {
    const tapir_query_grid& g = grids[i];
    TAPIR_CHECK_ARG(g.grid && g.out && g.h >= 1 && g.w >= 1 && g.C >= 1 &&
                        g.clip_stride >= (int64_t)g.h * g.w * g.C && aligned(g.grid, 4) && aligned(g.out, 4),
                    "%s: grid %d (%d x %d x %d, clip stride %lld) needs 4-byte aligned grid and out", fn, i,
                    g.h, g.w, g.C, (long long)g.clip_stride);
    TAPIR_CHECK_ARG(!overlap(g.out, (size_t)rows * g.C * 4, g.grid, (size_t)g.clip_stride * clips * 4),
                    "%s: grid %d's out overlaps its grid", fn, i);
  }
  return sample_query_rows(grids, num_grids, clips, rows, video_h, video_w, video_hw, count, requests,
                           state, num_state, S(stream));
}

size_t tapir_cost_volume_workspace_bytes(int32_t N, int32_t T, int32_t gh, int32_t gw, int32_t C) {
  return cost_volume_workspace_bytes(1, N, T, gh, gw, C);
}

size_t tapir_cost_volume_batched_workspace_bytes(int32_t B, int32_t N, int32_t T, int32_t gh,
                                                 int32_t gw, int32_t C) {
  return cost_volume_workspace_bytes(B, (long long)B * N, T, gh, gw, C);
}

int tapir_cost_volume_tracks(const tapir_head_weights* w, const float* qfeat, const float* grid,
                             int32_t N, int32_t T, int32_t gh, int32_t gw, int32_t C,
                             const float* query_tyx, float softmax_temperature, int32_t init_h,
                             int32_t init_w, float* points, float* occ, float* expd,
                             int32_t* argmax, void* workspace, size_t workspace_bytes,
                             void* stream) {
  Range nvtx_range("tapir_cost_volume_tracks");
  return cost_volume_tracks(w, qfeat, grid, 1, N, T, gh, gw, C, query_tyx, softmax_temperature,
                            init_h, init_w, points, occ, expd, argmax, workspace, workspace_bytes,
                            S(stream));
}

int tapir_cost_volume_tracks_batched(const tapir_head_weights* w, const float* qfeat,
                                     const float* grid, int32_t B, int32_t N, int32_t T, int32_t gh,
                                     int32_t gw, int32_t C, const float* query_tyx,
                                     float softmax_temperature, int32_t init_h, int32_t init_w,
                                     float* points, float* occ, float* expd, int32_t* argmax,
                                     void* workspace, size_t workspace_bytes, void* stream) {
  Range nvtx_range("tapir_cost_volume_tracks_batched");
  return cost_volume_tracks(w, qfeat, grid, B, N, T, gh, gw, C, query_tyx, softmax_temperature,
                            init_h, init_w, points, occ, expd, argmax, workspace, workspace_bytes,
                            S(stream));
}

size_t tapir_cost_volume_ragged_workspace_bytes(int32_t B, int32_t total_points, int32_t T, int32_t gh,
                                                int32_t gw, int32_t C) {
  return cost_volume_workspace_bytes(B, total_points, T, gh, gw, C);
}

int tapir_cost_volume_tracks_ragged(const tapir_head_weights* w, const float* qfeat, const float* grid,
                                    int32_t B, const int32_t* points_per_clip, int32_t T, int32_t gh,
                                    int32_t gw, int32_t C, const float* query_tyx,
                                    float softmax_temperature, int32_t init_h, int32_t init_w,
                                    float* points, float* occ, float* expd, int32_t* argmax,
                                    void* workspace, size_t workspace_bytes, void* stream) {
  Range nvtx_range("tapir_cost_volume_tracks_ragged");
  const char* fn = "tapir_cost_volume_tracks_ragged";
  TAPIR_CHECK_ARG(w && qfeat && grid && points && occ && expd && points_per_clip && workspace,
                  "%s: null pointer", fn);
  TAPIR_CHECK_ARG(B >= 1 && B <= TAPIR_MAX_RAGGED_CLIPS, "%s: B=%d clips, 1..%d supported", fn, B,
                  TAPIR_MAX_RAGGED_CLIPS);
  long long total = 0;
  for (int b = 0; b < B; ++b) {
    TAPIR_CHECK_ARG(points_per_clip[b] >= 1, "%s: clip %d has %d points", fn, b, points_per_clip[b]);
    total += points_per_clip[b];
  }
  TAPIR_CHECK_ARG(T >= 1 && gh >= 2 && gw >= 2 && C >= 64 && C % 64 == 0,
                  "%s: T=%d map %d x %d C=%d (T >= 1, maps at least 2 x 2, C a multiple of 64)", fn, T, gh,
                  gw, C);
  TAPIR_CHECK_ARG(total < (1ll << 31) && (long long)B * T * gh * gw < (1ll << 31),
                  "%s: %lld points over %d clips exceed one launch", fn, total, B);
  TAPIR_CHECK_ARG(init_h >= 1 && init_w >= 1, "%s: init_h=%d init_w=%d", fn, init_h, init_w);
  TAPIR_CHECK_ARG(aligned(qfeat, 16) && aligned(grid, 16), "%s: qfeat and grid must be 16-byte aligned", fn);
  const size_t need = cost_volume_workspace_bytes(B, total, T, gh, gw, C);
  TAPIR_CHECK_ARG(workspace_bytes >= need, "%s: workspace %zu bytes < %zu", fn, workspace_bytes, need);
  return cost_volume_tracks_ragged(w, qfeat, grid, B, points_per_clip, T, gh, gw, C, query_tyx,
                                   softmax_temperature, init_h, init_w, points, occ, expd, argmax,
                                   workspace, workspace_bytes, S(stream));
}

int tapir_pool_pyramid(const float* grid, int32_t T, int32_t h, int32_t w, int32_t C, float* out,
                       void* stream) {
  Range nvtx_range("tapir_pool_pyramid");
  TAPIR_CHECK_ARG(grid && out, "tapir_pool_pyramid: null pointer");
  TAPIR_CHECK_ARG(T > 0 && h >= 2 && w >= 2 && C > 0 && C % 4 == 0,
                  "tapir_pool_pyramid: T=%d h=%d w=%d C=%d (h, w >= 2, C a positive multiple of 4)", T, h, w, C);
  TAPIR_CHECK_ARG(aligned(grid, 16) && aligned(out, 16), "tapir_pool_pyramid: grid and out must be 16-byte aligned");
  return pool_pyramid(grid, T, h, w, C, out, S(stream));
}

// The correlation kernel reads the level grids and the query features as float4 and writes the
// output planes as bf16 pairs.
namespace {
int check_corr_args(const tapir_corr_args* a, int batch, const char* fn) {
  TAPIR_CHECK_ARG(a != nullptr && a->num_levels >= 1 && a->num_levels <= TAPIR_MAX_CORR_LEVELS,
                  "%s: bad level count", fn);
  TAPIR_CHECK_ARG(batch >= 1, "%s: bad clip count %d", fn, batch);
  TAPIR_CHECK_ARG(a->pos && a->occ && a->expd && a->feat_hi && a->feat_lo && a->out_planes, "%s: null pointer", fn);
  TAPIR_CHECK_ARG(a->init_h >= 1 && a->init_w >= 1, "%s: init_h=%d init_w=%d", fn, a->init_h, a->init_w);
  for (int l = 0; l < a->num_levels; ++l) {
    const tapir_corr_level& L = a->levels[l];
    TAPIR_CHECK_ARG(L.h >= 1 && L.w >= 1, "%s: level %d is %d x %d", fn, l, L.h, L.w);
    TAPIR_CHECK_ARG(aligned(L.grid, 16), "%s: level %d grid must be 16-byte aligned", fn, l);
  }
  TAPIR_CHECK_ARG(aligned(a->feat_hi, 16) && aligned(a->feat_lo, 16) && a->feat_hi_stride_n >= 0 &&
                      a->feat_hi_stride_t >= 0 && a->feat_lo_stride_n >= 0 && a->feat_lo_stride_t >= 0 &&
                      a->feat_hi_stride_n % 4 == 0 && a->feat_hi_stride_t % 4 == 0 &&
                      a->feat_lo_stride_n % 4 == 0 && a->feat_lo_stride_t % 4 == 0,
                  "%s: feat_hi, feat_lo must be 16-byte aligned, their strides non-negative multiples of 4", fn);
  TAPIR_CHECK_ARG(aligned(a->out_planes, 4) && a->out_plane_stride % 2 == 0,
                  "%s: out_planes must be 4-byte aligned, out_plane_stride even", fn);
  const long long rows = (long long)a->num_points * batch * a->num_frames;
  TAPIR_CHECK_ARG(a->planes <= 1 || a->out_plane_stride >= rows * a->ld,
                  "%s: planes overlap (out_plane_stride=%lld)", fn, (long long)a->out_plane_stride);
  return kOk;
}
}  // namespace

int tapir_local_corr(const tapir_corr_args* args, void* stream) {
  Range nvtx_range("tapir_local_corr");
  TAPIR_RETURN_IF(check_corr_args(args, 1, "tapir_local_corr"));
  return local_corr(args, 1, S(stream));
}

int tapir_local_corr_batched(const tapir_corr_args* args, int32_t batch, void* stream) {
  Range nvtx_range("tapir_local_corr_batched");
  TAPIR_RETURN_IF(check_corr_args(args, batch, "tapir_local_corr_batched"));
  return local_corr(args, batch, S(stream));
}

int tapir_local_corr_ragged(const tapir_corr_args* args, int32_t batch, const int32_t* query_clip,
                            void* stream) {
  Range nvtx_range("tapir_local_corr_ragged");
  const char* fn = "tapir_local_corr_ragged";
  TAPIR_RETURN_IF(check_corr_args(args, 1, fn));
  TAPIR_CHECK_ARG(batch >= 1, "%s: bad clip count %d", fn, batch);
  TAPIR_CHECK_ARG(query_clip != nullptr && aligned(query_clip, 4), "%s: query_clip must be a 4-byte aligned table",
                  fn);
  return local_corr(args, batch, S(stream), query_clip);
}

size_t tapir_mixer_workspace_bytes(int64_t rows, int32_t planes) {
  return mixer_workspace_bytes(rows, planes);
}

int tapir_mixer_forward(const tapir_mixer_weights* w, const tapir_mixer_io* io, void* workspace,
                        size_t workspace_bytes, void* stream) {
  Range nvtx_range("tapir_mixer_forward");
  return mixer_forward(w, io, workspace, workspace_bytes, S(stream));
}

int tapir_mixer_dw(const tapir_mixer_block* blk, const float* x, int32_t n, int32_t T, int32_t causal,
                   const float* ctx1_in, const float* ctx2_in, float* ctx1_out, float* ctx2_out, float* z,
                   void* planes_out, int64_t plane_stride, int32_t planes, void* stream) {
  Range nvtx_range("tapir_mixer_dw");
  TAPIR_CHECK_ARG(blk && x && z && planes_out, "tapir_mixer_dw: null pointer");
  TAPIR_CHECK_ARG(blk->ln_w && blk->dw1_w && blk->dw1_b && blk->dw2_w && blk->dw2_b && blk->ln1_w,
                  "tapir_mixer_dw: null weight pointer");
  TAPIR_CHECK_ARG(n >= 1 && n <= 65535 && T >= 1, "tapir_mixer_dw: n=%d T=%d (n in 1..65535, T >= 1)", n, T);
  TAPIR_CHECK_ARG(planes >= 1 && planes <= 3, "tapir_mixer_dw: planes=%d", planes);
  const long long rows = (long long)n * T;
  TAPIR_CHECK_ARG(planes == 1 || plane_stride >= rows * 512,
                  "tapir_mixer_dw: planes overlap (plane_stride=%lld)", (long long)plane_stride);
  TAPIR_CHECK_ARG(aligned(x, 16) && aligned(z, 16) && aligned(ctx1_in, 16) && aligned(ctx2_in, 16) &&
                      aligned(ctx1_out, 16) && aligned(ctx2_out, 16) && aligned(blk->ln_w, 16) &&
                      aligned(blk->ln1_w, 16) && aligned(planes_out, 8) && plane_stride % 4 == 0,
                  "tapir_mixer_dw: x, z, contexts and LayerNorm weights must be 16-byte aligned, "
                  "planes_out 8-byte aligned, plane_stride a multiple of 4");
  TAPIR_CHECK_ARG(!overlap(x, rows * 512 * 4, z, rows * 512 * 4), "tapir_mixer_dw: x and z overlap");
  TAPIR_CHECK_ARG(causal || !(ctx1_in || ctx2_in || ctx1_out || ctx2_out),
                  "tapir_mixer_dw: context pointers on a non-causal call");
  // T > 24 runs several CTAs per query: one would read a context slot another has overwritten.
  // T = 1 reads both slots before writing (the streaming step updates its context in place).
  const size_t c1 = (size_t)n * 2 * 512 * 4, c2 = (size_t)n * 2 * 2048 * 4;
  TAPIR_CHECK_ARG(!overlap(ctx1_in, ctx1_in ? c1 : 0, ctx1_out, ctx1_out ? c1 : 0) ||
                      (T == 1 && ctx1_in == ctx1_out),
                  "tapir_mixer_dw: ctx1_in and ctx1_out overlap (allowed only as the same buffer at T = 1)");
  TAPIR_CHECK_ARG(!overlap(ctx2_in, ctx2_in ? c2 : 0, ctx2_out, ctx2_out ? c2 : 0) ||
                      (T == 1 && ctx2_in == ctx2_out),
                  "tapir_mixer_dw: ctx2_in and ctx2_out overlap (allowed only as the same buffer at T = 1)");
  return mixer_dw(*blk, x, n, T, causal != 0, ctx1_in, ctx2_in, ctx1_out, ctx2_out, z,
                  static_cast<__nv_bfloat16*>(planes_out), plane_stride, planes, S(stream));
}

namespace {
int check_update_args(const tapir_update_args* a, bool per_clip_video, const char* who) {
  TAPIR_CHECK_ARG(a != nullptr && a->res && a->pos && a->feat_out && a->occ_out && a->expd_out && a->feat_hi &&
                      a->feat_lo && a->occ_in && a->expd_in,
                  "%s: null pointer", who);
  const long long rows = (long long)a->num_points * a->num_frames;
  TAPIR_CHECK_ARG(a->num_points >= 1 && a->num_frames >= 1 && rows < (1ll << 31),
                  "%s: num_points=%d num_frames=%d (rows must be in 1..2^31-1)", who, a->num_points,
                  a->num_frames);
  TAPIR_CHECK_ARG(a->ld_res >= 388, "%s: ld_res=%d < 388", who, a->ld_res);
  TAPIR_CHECK_ARG(a->init_h >= 1 && a->init_w >= 1 && a->resize_h >= 1 && a->resize_w >= 1 &&
                      (a->tracks_out == nullptr || per_clip_video || (a->video_h >= 1 && a->video_w >= 1)),
                  "%s: sizes must be positive", who);
  return kOk;
}
}  // namespace

int tapir_refine_update(const tapir_update_args* args, void* stream) {
  Range nvtx_range("tapir_refine_update");
  TAPIR_RETURN_IF(check_update_args(args, false, "tapir_refine_update"));
  return refine_update(args, S(stream));
}

int tapir_refine_update_ex(const tapir_update_args* args, const int32_t* video_hw,
                           int32_t rows_per_clip, void* stream) {
  Range nvtx_range("tapir_refine_update_ex");
  if (video_hw == nullptr) return tapir_refine_update(args, stream);
  TAPIR_RETURN_IF(check_update_args(args, true, "tapir_refine_update_ex"));
  const long long rows = (long long)args->num_points * args->num_frames;
  TAPIR_CHECK_ARG(args->tracks_out != nullptr, "tapir_refine_update_ex: a video size table needs tracks_out");
  TAPIR_CHECK_ARG(rows_per_clip >= 1 && rows % rows_per_clip == 0 && rows_per_clip % args->num_frames == 0,
                  "tapir_refine_update_ex: rows_per_clip=%d does not divide the %lld rows into clips of "
                  "whole queries (%d frames each)", rows_per_clip, rows, args->num_frames);
  TAPIR_CHECK_ARG((reinterpret_cast<uintptr_t>(video_hw) & 3) == 0,
                  "tapir_refine_update_ex: video_hw not 4-byte aligned");
  return refine_update(args, S(stream), video_hw, rows_per_clip);
}

int tapir_refine_update_ragged(const tapir_update_args* args, const int32_t* video_hw,
                               const int32_t* query_clip, void* stream) {
  Range nvtx_range("tapir_refine_update_ragged");
  const char* fn = "tapir_refine_update_ragged";
  TAPIR_RETURN_IF(check_update_args(args, true, fn));
  TAPIR_CHECK_ARG(args->tracks_out != nullptr, "%s: a video size table needs tracks_out", fn);
  TAPIR_CHECK_ARG(video_hw != nullptr && query_clip != nullptr && aligned(video_hw, 4) && aligned(query_clip, 4),
                  "%s: video_hw and query_clip must be 4-byte aligned device tables", fn);
  return refine_update(args, S(stream), video_hw, 0, query_clip);
}

size_t tapir_paint_point_track_workspace_bytes(int32_t frames, int32_t points) {
  return paint_point_track_workspace_bytes(frames, points);
}

int tapir_paint_point_track(const uint8_t* frames, int32_t T, int32_t H, int32_t W, const void* tracks,
                            int32_t tracks_fp64, const uint8_t* visibles, int32_t N, const uint8_t* colors,
                            uint8_t* out, void* workspace, size_t workspace_bytes, void* stream) {
  Range nvtx_range("tapir_paint_point_track");
  TAPIR_CHECK_ARG(T >= 0 && H >= 0 && W >= 0 && N >= 0,
                  "tapir_paint_point_track: negative size (T=%d H=%d W=%d N=%d)", T, H, W, N);
  TAPIR_CHECK_ARG(tracks_fp64 == 0 || tracks_fp64 == 1, "tapir_paint_point_track: tracks_fp64=%d", tracks_fp64);
  const long long tiles_per_frame = ((H + 31ll) / 32) * ((W + 31ll) / 32);
  TAPIR_CHECK_ARG(tiles_per_frame == 0 || T <= INT32_MAX / tiles_per_frame,
                  "tapir_paint_point_track: %d frames of %d x %d exceed one launch grid", T, H, W);
  const long long pixels = (long long)T * H * W;
  if (pixels == 0) return kOk;
  TAPIR_CHECK_ARG(frames && out, "tapir_paint_point_track: null frames / out");
  TAPIR_CHECK_ARG(!overlap(frames, (size_t)pixels * 3, out, (size_t)pixels * 3),
                  "tapir_paint_point_track: out overlaps frames (painting is not in place)");
  if (N > 0) {
    TAPIR_CHECK_ARG(tracks && visibles && colors && workspace, "tapir_paint_point_track: null pointer");
    TAPIR_CHECK_ARG(aligned(tracks, tracks_fp64 ? 8 : 4) && aligned(workspace, 16),
                    "tapir_paint_point_track: tracks must be aligned to their dtype, workspace 16-byte aligned");
    const size_t need = paint_point_track_workspace_bytes(T, N);
    TAPIR_CHECK_ARG(workspace_bytes >= need, "tapir_paint_point_track: workspace %zu bytes < %zu",
                    workspace_bytes, need);
  }
  return paint_point_track(frames, T, H, W, tracks, tracks_fp64, visibles, N, colors, out, workspace,
                           S(stream));
}

int tapir_ransac_stop_thresholds(int32_t N, double targ_inlier_frac, double* out) {
  TAPIR_CHECK_ARG(N >= 1 && out != nullptr, "tapir_ransac_stop_thresholds: N=%d, out %p", N, (void*)out);
  TAPIR_CHECK_ARG(std::isfinite(targ_inlier_frac) && targ_inlier_frac > 0.0,
                  "tapir_ransac_stop_thresholds: targ_inlier_frac=%g must be positive", targ_inlier_frac);
  ransac_stop_thresholds(N, targ_inlier_frac, out);
  return kOk;
}

size_t tapir_homographies_workspace_bytes(int32_t T, int32_t N) {
  return homographies_workspace_bytes(T, N);
}

int tapir_homographies_wrt_frame(const tapir_homography_args* a, void* stream) {
  Range nvtx_range("tapir_homographies_wrt_frame");
  const char* fn = "tapir_homographies_wrt_frame";
  TAPIR_CHECK_ARG(a != nullptr, "%s: null args", fn);
  TAPIR_CHECK_ARG(a->N >= 1 && a->T >= 1 && (long long)a->N * a->T <= (1ll << 30),
                  "%s: bad shape N=%d T=%d (N, T >= 1, N T <= 2^30)", fn, a->N, a->T);
  TAPIR_CHECK_ARG(a->tracks_fp64 == 0 || a->tracks_fp64 == 1, "%s: tracks_fp64=%d", fn, a->tracks_fp64);
  TAPIR_CHECK_ARG(a->reference_frame >= 0 && a->reference_frame < a->T,
                  "%s: reference_frame=%d outside 0..%d", fn, a->reference_frame, a->T - 1);
  TAPIR_CHECK_ARG(std::isfinite(a->width) && std::isfinite(a->height) && a->width > 0 && a->height > 0,
                  "%s: image size %g x %g must be positive", fn, a->width, a->height);
  TAPIR_CHECK_ARG(std::isfinite(a->thresh) && a->thresh > 0 && std::isfinite(a->outlier_point_threshold) &&
                      a->outlier_point_threshold > 0,
                  "%s: thresh=%g and outlier_point_threshold=%g must be positive", fn, a->thresh,
                  a->outlier_point_threshold);
  TAPIR_CHECK_ARG(a->num_refinement_passes >= 0 && a->num_refinement_passes <= 1000,
                  "%s: num_refinement_passes=%d outside 0..1000", fn, a->num_refinement_passes);
  TAPIR_CHECK_ARG(a->tracks && a->occluded && a->stop_thresholds && a->homogs && a->err && a->canonical &&
                      a->workspace,
                  "%s: null pointer", fn);
  TAPIR_CHECK_ARG(aligned(a->tracks, a->tracks_fp64 ? 8 : 4) && aligned(a->stop_thresholds, 8) &&
                      aligned(a->homogs, 8) && aligned(a->err, 8) && aligned(a->canonical, 8) &&
                      aligned(a->ransac_stats, 4) && aligned(a->workspace, 256),
                  "%s: tracks and outputs must be aligned to their dtype, workspace to 256 bytes", fn);
  const size_t need = homographies_workspace_bytes(a->T, a->N);
  TAPIR_CHECK_ARG(a->workspace_bytes >= need, "%s: workspace %zu bytes < %zu", fn, a->workspace_bytes, need);
  return homographies_wrt_frame(a, S(stream));
}

namespace {
bool resize_side_ok(int n) { return n >= 1 && n <= TAPIR_MAX_RESIZE_SIDE; }
}  // namespace

int32_t tapir_lanczos_weights(int32_t in_size, int32_t out_size, int32_t* bounds, int32_t* taps) {
  if (!resize_side_ok(in_size) || !resize_side_ok(out_size)) {
    set_error("tapir_lanczos_weights: sizes %d -> %d outside 1..%d", in_size, out_size,
              TAPIR_MAX_RESIZE_SIDE);
    return -1;
  }
  if (bounds != nullptr && taps != nullptr) lanczos_weights(in_size, out_size, bounds, taps);
  return lanczos_ksize(in_size, out_size);
}

size_t tapir_resize_lanczos_u8_workspace_bytes(int32_t frames, int32_t H, int32_t W, int32_t h,
                                               int32_t w) {
  if (frames < 1 || !resize_side_ok(H) || !resize_side_ok(W) || !resize_side_ok(h) || !resize_side_ok(w))
    return 0;
  return resize_lanczos_u8_workspace_bytes(frames, H, W, h, w);
}

int tapir_resize_lanczos_u8(const uint8_t* src, uint8_t* dst, int32_t frames, int32_t H, int32_t W,
                            int32_t h, int32_t w, const int32_t* x_bounds, const int32_t* x_taps,
                            int32_t x_ksize, const int32_t* y_bounds, const int32_t* y_taps,
                            int32_t y_ksize, void* workspace, size_t workspace_bytes, void* stream) {
  Range nvtx_range("tapir_resize_lanczos_u8");
  const char* fn = "tapir_resize_lanczos_u8";
  TAPIR_CHECK_ARG(frames >= 1 && resize_side_ok(H) && resize_side_ok(W) && resize_side_ok(h) &&
                      resize_side_ok(w),
                  "%s: frames=%d %dx%d -> %dx%d (frames >= 1, sides in 1..%d)", fn, frames, H, W, h, w,
                  TAPIR_MAX_RESIZE_SIDE);
  TAPIR_CHECK_ARG(src && dst, "%s: null src / dst", fn);
  const size_t src_bytes = (size_t)frames * H * W * 3, dst_bytes = (size_t)frames * h * w * 3;
  TAPIR_CHECK_ARG(!overlap(src, src_bytes, dst, dst_bytes), "%s: dst overlaps src", fn);
  if (W != w) {
    TAPIR_CHECK_ARG(x_bounds && x_taps && aligned(x_bounds, 4) && aligned(x_taps, 4),
                    "%s: width %d -> %d needs the x tables (4-byte aligned)", fn, W, w);
    TAPIR_CHECK_ARG(x_ksize == lanczos_ksize(W, w), "%s: x_ksize=%d, the %d -> %d tables have %d taps",
                    fn, x_ksize, W, w, lanczos_ksize(W, w));
  }
  if (H != h) {
    TAPIR_CHECK_ARG(y_bounds && y_taps && aligned(y_bounds, 4) && aligned(y_taps, 4),
                    "%s: height %d -> %d needs the y tables (4-byte aligned)", fn, H, h);
    TAPIR_CHECK_ARG(y_ksize == lanczos_ksize(H, h), "%s: y_ksize=%d, the %d -> %d tables have %d taps",
                    fn, y_ksize, H, h, lanczos_ksize(H, h));
  }
  const size_t need = resize_lanczos_u8_workspace_bytes(frames, H, W, h, w);
  if (need > 0) {
    TAPIR_CHECK_ARG(workspace && aligned(workspace, 16), "%s: workspace must be non-NULL and 16-byte aligned", fn);
    TAPIR_CHECK_ARG(workspace_bytes >= need, "%s: workspace %zu bytes < %zu", fn, workspace_bytes, need);
    TAPIR_CHECK_ARG(!overlap(workspace, need, src, src_bytes) && !overlap(workspace, need, dst, dst_bytes),
                    "%s: workspace overlaps src or dst", fn);
  }
  return resize_lanczos_u8(src, dst, frames, H, W, h, w, x_bounds, x_taps, x_ksize, y_bounds, y_taps,
                           y_ksize, static_cast<uint8_t*>(workspace), S(stream));
}

}  // extern "C"
