/* tapir_b200 - C ABI of the B200-native TAPIR / BootsTAPIR inference hot path.
 *
 * The reference (google-deepmind/tapnet) has no FFI: its boundary is the Python class
 * tapnet/torch/tapir_model.py:TAPIR.  These entry points are what a C-ABI replacement of that
 * class's stages binds (SURVEY.md section 8(b)); each cites the reference code it replaces.
 *
 * Conventions
 *  - every pointer is a DEVICE pointer unless marked "host"; tensors are dense, channel-last,
 *    fp32 unless stated; "planes" are bf16 [P][rows][ld] split representations (x = p0+p1(+p2)).
 *  - `stream` is a cudaStream_t passed as void*; calls are asynchronous w.r.t. the host and
 *    never allocate, free or retain pointers; scratch comes from the caller (`workspace`,
 *    sized by the matching *_workspace_bytes).
 *  - return 0 on success; non-zero = error (1 bad argument, 2 unsupported, 3 CUDA error,
 *    4 workspace too small) with a message available from tapir_last_error() (thread local).
 *  - no CPU fallback exists: without a CUDA device every compute entry point fails.
 */
#ifndef TAPIR_B200_H_
#define TAPIR_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TAPIR_B200_ABI_VERSION 2 /* 2: TAPIR_MAX_CORR_LEVELS 3 -> 5 (tapir_corr_args grew) */
#define TAPIR_MAX_MIXER_BLOCKS 12
#define TAPIR_NUM_RESNET_BLOCKS 8
#define TAPIR_MAX_EXTRA_BLOCKS 5
#define TAPIR_MAX_CORR_LEVELS 5 /* hires + lowres + up to 3 pooled levels (pyramid_level <= 3) */
#define TAPIR_MAX_RAGGED_CLIPS 64 /* clips of one tapir_cost_volume_tracks_ragged call */

/* A dense layer / convolution prepared for the split-bf16 tensor-core GEMM:
 * w = bf16 planes [planes][N][K] (K padded with zeros to a multiple of 64; for 3x3
 * convolutions K is ordered (ky, kx, cin)), bias fp32 [N] or NULL. */
typedef struct tapir_linear {
  const void* w;
  const float* bias;
  int32_t N;
  int32_t K;
  int32_t planes;
  int32_t k_logical; /* un-padded contraction length (profiling only; 0 = K) */
} tapir_linear;

/* nets.py:247-327 BlockV2 (InstanceNorm affine eps 1e-5). */
typedef struct tapir_resnet_block {
  tapir_linear proj;  /* 1x1, only when has_proj */
  tapir_linear conv0; /* 3x3, stride `stride` */
  tapir_linear conv1; /* 3x3, stride 1 */
  const float* bn0_w;
  const float* bn0_b;
  const float* bn1_w;
  const float* bn1_b;
  int32_t cin, cout, stride, has_proj;
} tapir_resnet_block;

/* nets.py:25-62 ExtraConvBlock. */
typedef struct tapir_extra_block {
  const float* ln_w;
  const float* ln_b;
  tapir_linear conv;   /* 3x3 256 -> 1024 (+bias, tanh-GELU) */
  tapir_linear conv1;  /* 3x3 1024 -> 256 (+bias) */
} tapir_extra_block;

typedef struct tapir_backbone_weights {
  const float* stem_w; /* [7][7][3][64] fp32 (ky,kx,cin,cout) repack of initial_conv.weight */
  tapir_resnet_block blocks[TAPIR_NUM_RESNET_BLOCKS];
  tapir_extra_block extra[TAPIR_MAX_EXTRA_BLOCKS];
  int32_t num_extra; /* 0 when extra_convs=False */
  int32_t planes;    /* split-bf16 planes used for activations (1..3) */
} tapir_backbone_weights;

/* tapir_model.py:121-127 torch_cost_volume_track_mods; all fp32, torch layouts. */
typedef struct tapir_head_weights {
  const float* hid1_w; /* [16][1][3][3] */
  const float* hid1_b;
  const float* hid2_w; /* [1][16][3][3] */
  const float* hid2_b;
  const float* hid3_w; /* [32][16][3][3] */
  const float* hid3_b;
  const float* hid4_w; /* [16][32] */
  const float* hid4_b;
  const float* occ_w;  /* [2][16] */
  const float* occ_b;
} tapir_head_weights;

/* nets.py:107-186 PIPsConvBlock. dw*_w are the torch Conv1d weights [2048][1][3]. */
typedef struct tapir_mixer_block {
  const float* ln_w;
  const float* dw1_w;
  const float* dw1_b;
  const float* dw2_w;
  const float* dw2_b;
  const float* ln1_w;
  tapir_linear up;   /* 512 -> 2048 (+bias, tanh-GELU) */
  tapir_linear down; /* 2048 -> 512 (+bias) */
} tapir_mixer_block;

/* nets.py:189-244 PIPSMLPMixer. */
typedef struct tapir_mixer_weights {
  tapir_linear linear;   /* in_dim (padded to 64) -> 512 */
  tapir_linear linear_1; /* 512 -> 388 */
  const float* ln_w;
  tapir_mixer_block blocks[TAPIR_MAX_MIXER_BLOCKS];
  int32_t num_blocks;
  int32_t planes;
} tapir_mixer_weights;

typedef struct tapir_mixer_io {
  const void* x_planes;    /* bf16 [planes][rows][ldx]: mixer input rows (n-major, t-minor) */
  int64_t x_plane_stride;  /* elements */
  int32_t ldx;
  int32_t num_points;      /* n */
  int32_t num_frames;      /* T ; rows = n*T */
  int32_t causal;          /* use_casual_conv */
  /* causal context (nets.py:149-176), host arrays of num_blocks device pointers, each fp32
   * [n][2][512] (ctx1) / [n][2][2048] (ctx2); all NULL = zero context / not requested */
  const float* const* ctx1_in;
  const float* const* ctx2_in;
  float* const* ctx1_out;
  float* const* ctx2_out;
  float* out;              /* fp32 [rows][ldo] ; first 388 columns valid */
  int32_t ldo;
  int32_t reserved;
} tapir_mixer_io;

typedef struct tapir_corr_level {
  const float* grid; /* [T][h][w][C] fp32, L2-normalised features */
  int32_t h, w, C, reserved;
} tapir_corr_level;

/* tapir_model.py:599-658: local correlation + assembly of the mixer input row. */
typedef struct tapir_corr_args {
  tapir_corr_level levels[TAPIR_MAX_CORR_LEVELS];
  int32_t num_levels;    /* 2 + pyramid_level */
  int32_t num_points;    /* n */
  int32_t num_frames;    /* T */
  int32_t init_h, init_w;/* coordinate frame of `pos` (initial_resolution) */
  int32_t planes;
  const float* pos;      /* [n][T][2] (x,y) */
  const float* occ;      /* [n][T] */
  const float* expd;     /* [n][T] */
  /* 128-ch (hires) and 256-ch (lowres) halves of the per-row feature: element (i,t,c) at
   * ptr[i*stride_n + t*stride_t + c]; stride_t = 0 broadcasts a per-query feature. */
  const float* feat_hi;
  int64_t feat_hi_stride_n, feat_hi_stride_t;
  const float* feat_lo;
  int64_t feat_lo_stride_n, feat_lo_stride_t;
  void* out_planes;      /* bf16 [planes][n*T][ld] */
  int64_t out_plane_stride;
  int32_t ld;            /* >= 388 + 49*num_levels, multiple of 64; pad columns are zeroed */
  int32_t reserved;
} tapir_corr_args;

/* tapir_model.py:674-685 + train2orig :435-441. */
typedef struct tapir_update_args {
  const float* res;      /* mixer output [n*T][ld_res] */
  int32_t ld_res;
  int32_t num_points, num_frames;
  int32_t init_h, init_w;       /* initial_resolution */
  int32_t resize_h, resize_w;   /* refinement resolution of this level */
  int32_t video_h, video_w;     /* original video size (for tracks_out) */
  int32_t reserved;
  const float* feat_hi;
  int64_t feat_hi_stride_n, feat_hi_stride_t;
  const float* feat_lo;
  int64_t feat_lo_stride_n, feat_lo_stride_t;
  float* pos;            /* [n][T][2] in/out (initial_resolution pixels) */
  const float* occ_in;   /* [n][T] */
  const float* expd_in;
  float* occ_out;        /* [n][T] (may alias occ_in) */
  float* expd_out;
  float* feat_out;       /* [n][T][384] = res[4:] + feat */
  float* tracks_out;     /* [n][T][2] pos scaled to the video size, or NULL */
} tapir_update_args;

/* ---- library ---------------------------------------------------------------------- */
const char* tapir_last_error(void);
int tapir_abi_version(void);
/* kernels launched by this library since load (bench.py reports it as gpu_launches) */
unsigned long long tapir_launch_count(void);

/* Per-launch device timing (CUDA events on the launch stream).  tapir_profile_report
 * synchronises the device, writes a JSON object {"kernel class": {"launches", "ms", "flops",
 * "bytes"}} (algorithmic flops / bytes per SURVEY.md 8(d)) into buf and clears the records. */
void tapir_profile_enable(int32_t on);
int tapir_profile_report(char* buf, size_t capacity);

/* fp32 [rows][ld_src] -> bf16 planes [planes][rows][ld_dst]; columns cols..cols_padded-1 are
 * zero filled.  Used to prepare weights and features for the GEMMs. */
int tapir_split_planes(const float* src, int64_t ld_src, void* dst, int64_t ld_dst,
                       int64_t plane_stride, int64_t rows, int32_t cols, int32_t cols_padded,
                       int32_t planes, void* stream);

/* Generic split-bf16 GEMM  out = act(A . B^T + bias) + residual  (see csrc/gemm.cuh).
 * impl: 0 = tcgen05 (product path), 1 = SIMT cross-check. conv3x3 != 0 treats A as NHWC
 * planes [planes][frames][H][W][C] (stride 1, zero padding 1).  stats (nullable): fp64
 * [frames][N][2] accumulators that receive the per-(frame, column) sum and sum of squares of
 * the output (the InstanceNorm statistics of the produced tensor); the caller zeroes them. */
int tapir_gemm(const void* a_planes, int32_t lda, int64_t a_plane_stride, const tapir_linear* b,
               int64_t M, int32_t conv3x3, int32_t frames, int32_t H, int32_t W, int32_t C,
               const float* residual, int32_t ldr, int32_t act_gelu, float* out_f32, int32_t ldo,
               void* out_planes, int32_t ldp, int64_t out_plane_stride, int32_t out_P,
               double* stats, int32_t rows_per_frame, int32_t impl, void* stream);

/* tapir_gemm plus a split-K scratch buffer.  A non-NULL `splitk_workspace` lets the wgmma path
 * split K over several CTAs when the problem cannot fill the GPU (K >= 2048, no stats): raw fp32
 * partial sums go to the workspace and a second kernel sums them in a fixed order and applies the
 * epilogue.  The split count shrinks until S * M * round_up(N, 8) floats fit in
 * `splitk_workspace_bytes`; if no split fits, the GEMM runs in one pass.  This is what the
 * single-frame (streaming) mixer and backbone calls do; the summation order then depends on M. */
int tapir_gemm_ex(const void* a_planes, int32_t lda, int64_t a_plane_stride, const tapir_linear* b,
                  int64_t M, int32_t conv3x3, int32_t frames, int32_t H, int32_t W, int32_t C,
                  const float* residual, int32_t ldr, int32_t act_gelu, float* out_f32,
                  int32_t ldo, void* out_planes, int32_t ldp, int64_t out_plane_stride,
                  int32_t out_P, double* stats, int32_t rows_per_frame, int32_t impl,
                  void* splitk_workspace, size_t splitk_workspace_bytes, void* stream);

/* ---- a3: tapir_model.py:293-392 get_feature_grids (one resolution, one frame chunk) ---- */
/* utils.py:26-42 bilinear resize, align_corners=False, [frames][H][W][C] -> [frames][oH][oW][C] */
int tapir_bilinear_resize(const float* src, int32_t frames, int32_t H, int32_t W, int32_t C,
                          float* dst, int32_t oH, int32_t oW, void* stream);

/* The backbone's memory-bound building blocks, one kernel each (what tapir_backbone_forward runs
 * around its GEMMs).  Every argument is checked before any CUDA call: a NULL pointer, an
 * unsupported C, planes outside 1..3, frames above 65535 (where frames run on a grid dimension)
 * or a pointer / plane stride misaligned for the kernel's vector accesses returns 1.  Planes are
 * bf16 [planes][...] at `plane_stride` elements, each the fp32 residual of the ones before. */
/* nets.py:395-402,420: F.pad(x, (2, 4, 2, 4)) then the 7x7 stride-2 conv 3 -> 64, no bias.
 * video [frames][H][W][3] fp32 in [-1,1], or uint8 [0,255] when video_u8 != 0 (normalised as
 * x / 255 * 2 - 1 in fp32, each operation rounded); H, W even; w_packed [7][7][3][64] is
 * initial_conv.weight.permute(2, 3, 1, 0); out [frames][H/2][W/2][64]. */
int tapir_stem_conv(const void* video, int32_t video_u8, const float* w_packed, int32_t frames,
                    int32_t H, int32_t W, float* out, void* stream);
/* InstanceNorm statistics of x [frames][hw][C], C in {64, 128, 256}: sums [frames][C][2] fp64
 * (sum, sum of squares), zeroed by the call, then accumulated in fp64. */
int tapir_instnorm_stats(const float* x, int32_t frames, int64_t hw, int32_t C, double* sums,
                         void* stream);
/* nets.py:280-286,315-316: relu(InstanceNorm(x) * w + b) (biased variance, eps 1e-5) from the
 * sums of tapir_instnorm_stats, split into `planes` bf16 planes [frames][hw][C].  zero_next
 * (nullable) receives 0.0 in its first frames * 2 * zero_channels doubles. */
int tapir_instnorm_relu_split(const float* x, const double* sums, const float* w, const float* b,
                              int32_t frames, int64_t hw, int32_t C, void* out_planes,
                              int64_t plane_stride, int32_t planes, double* zero_next,
                              int32_t zero_channels, void* stream);
/* nets.py:258-267,320: the rows of a stride-2 conv over F.pad(x, (0, 2, 0, 2)).  in_planes
 * [planes][frames][H][W][C] bf16 (H, W even, C % 8 == 0) -> out_planes
 * [planes][frames][H/2][W/2][taps][C]; taps 9: tap (ky, kx) = ky * 3 + kx reads
 * in[2y + ky][2x + kx] (zero outside), taps 1: in[2y][2x]. */
int tapir_im2col_s2(const void* in_planes, int64_t in_plane_stride, int32_t frames, int32_t H,
                    int32_t W, int32_t C, int32_t taps, void* out_planes, int64_t out_plane_stride,
                    int32_t planes, void* stream);
/* LayerNorm over the last dimension (eps 1e-5), C in {256, 512}: x [rows][C] -> y [rows][C]
 * fp32 (nullable) and / or `planes` bf16 planes [rows][C] (planes_out nullable); b nullable
 * (nets.py:37-39,56 with bias, :118-120,138-140 without). */
int tapir_layernorm_split(const float* x, int64_t rows, int32_t C, const float* w, const float* b,
                          float* y, void* planes_out, int64_t plane_stride, int32_t planes,
                          void* stream);
/* tapir_model.py:370-381: x / sqrt(max(sum x^2, 1e-12)) per row, C in {128, 256}. */
int tapir_l2_normalize(const float* x, int64_t rows, int32_t C, float* out, void* stream);
size_t tapir_backbone_workspace_bytes(int32_t frames, int32_t H, int32_t W, int32_t extra_convs,
                                      int32_t planes);
/* video [frames][H][W][3] in [-1,1] -> lowres [frames][H/8][W/8][256], hires
 * [frames][H/4][W/4][128], both L2-normalised over channels (nets.py ResNet + ExtraConvs). */
int tapir_backbone_forward(const tapir_backbone_weights* w, const float* video, int32_t frames,
                           int32_t H, int32_t W, float* lowres, float* hires, void* workspace,
                           size_t workspace_bytes, void* stream);

/* Same, reading raw uint8 [0,255] frames: preprocess_frames (pytorch_live_demo.py:30-41,
 * x / 255 * 2 - 1) is applied inside the stem conv's loads, the float video never exists. */
int tapir_backbone_forward_u8(const tapir_backbone_weights* w, const uint8_t* video,
                              int32_t frames, int32_t H, int32_t W, float* lowres, float* hires,
                              void* workspace, size_t workspace_bytes, void* stream);

/* Same two calls with one more argument: `hires_ready_event` (a cudaEvent_t as void*, or NULL)
 * is recorded on `stream` as soon as the hires output is final, i.e. before ResNet groups 2-3
 * and the ExtraConvs run.  The multi-GPU path (SURVEY.md 8(e)) starts the all-gather of the hires
 * grid on another stream at that point, hidden behind the rest of the backbone.  video_u8 != 0
 * selects the uint8 reader. */
int tapir_backbone_forward_ex(const tapir_backbone_weights* w, const void* video, int32_t video_u8,
                              int32_t frames, int32_t H, int32_t W, float* lowres, float* hires,
                              void* workspace, size_t workspace_bytes, void* hires_ready_event,
                              void* stream);

/* Host-resident clips: the stem convolution (the only reader of the video) of frames
 * [frame0, frame0 + nframes) of a `pass_frames`-frame backbone pass, run as soon as that chunk
 * has arrived over PCIe while later chunks are still in flight.  `video_chunk` points at frame
 * `frame0`.  After every frame of the pass has been through this call (same workspace, same
 * pass_frames / H / W), tapir_backbone_forward_ex with video == NULL runs the rest. */
int tapir_backbone_stem(const tapir_backbone_weights* w, const void* video_chunk, int32_t video_u8,
                        int32_t pass_frames, int32_t H, int32_t W, int32_t frame0, int32_t nframes,
                        void* workspace, size_t workspace_bytes, void* stream);

/* ---- SURVEY 8f row 1: frame ingest (the step before the path) ------------------------ */
/* uint8 frames [frames][H][W][3] -> crop window (get_frame's centre square crop,
 * pytorch_live_demo.py:88-95, or any window) -> preprocess_frames (:30-41) -> utils.bilinear
 * (utils.py:26-42) to [frames][oH][oW][3] float in [-1,1]; one pass. */
int tapir_ingest_frames(const uint8_t* src, int32_t frames, int32_t H, int32_t W, int32_t crop_y,
                        int32_t crop_x, int32_t crop_h, int32_t crop_w, float* dst, int32_t oH,
                        int32_t oW, void* stream);

/* 8-bit YUV 4:2:0 frames as video decoders (NV12) and cameras (NV12 / I420) deliver them.
 * Luma sample (r, c) of frame f is y[f * y_frame_stride + r * y_pitch + c]; chroma sample
 * (r, c) is u[f * u_frame_stride + r * u_pitch + c * chroma_step] (v likewise), with chroma
 * planes of ceil(H/2) x ceil(W/2) samples.  I420: chroma_step 1; NV12: chroma_step 2 and
 * v = u + 1 (the interleaved UV plane).  Strides and pitches are in bytes.
 *
 * Conversion contract: pixel (r, c) of the full frame uses chroma sample (r >> 1, c >> 1)
 * (nearest, no interpolation; a crop window keeps absolute coordinates).  With D = U - 128,
 * E = V - 128 and C = Y - 16, k = 298 (limited range) or C = Y, k = 256 (full range):
 *   R = (k*C + cr*E + 128) >> 8, G = (k*C - gu*D - gv*E + 128) >> 8, B = (k*C + bu*D + 128) >> 8
 * (arithmetic shift, then clamped to [0, 255]), where (cr, gu, gv, bu) is
 *   BT.601 limited (409, 100, 208, 516)   BT.709 limited (459, 55, 136, 541)
 *   BT.601 full    (359,  88, 183, 454)   BT.709 full    (403, 48, 120, 475).
 * Everything after that is the uint8 RGB path (x / 255 * 2 - 1, each operation rounded), so a
 * YUV frame gives bit for bit the results of the uint8 RGB frame the conversion produces. */
typedef struct tapir_yuv420_frames {
  const uint8_t* y;
  const uint8_t* u;
  const uint8_t* v;
  int64_t y_frame_stride, u_frame_stride, v_frame_stride;
  int64_t y_pitch, u_pitch, v_pitch;
  int32_t chroma_step;     /* 1 (I420) or 2 (NV12) */
  int32_t H, W;            /* full frame (luma samples) */
  int32_t y0, x0, h, w;    /* crop window inside the frame */
  int32_t matrix;          /* 601 or 709 */
  int32_t full_range;      /* 0: limited (16-235 luma), 1: full (0-255) */
  int32_t reserved;
} tapir_yuv420_frames;

/* Crop window of `frames` frames -> uint8 RGB [frames][h][w][3] (dense). */
int tapir_yuv420_to_rgb(const tapir_yuv420_frames* src, int32_t frames, uint8_t* dst, void* stream);

/* tapir_ingest_frames for YUV 4:2:0: crop window -> RGB -> [-1,1] -> bilinear resize to
 * [frames][oH][oW][3] float, one pass; each of the four taps is converted, then the uint8
 * arithmetic runs unchanged. */
int tapir_ingest_frames_yuv420(const tapir_yuv420_frames* src, int32_t frames, float* dst,
                               int32_t oH, int32_t oW, void* stream);

/* YUV frames of any common decoder or camera layout: 8- to 16-bit samples, 4:2:0, 4:2:2 or 4:4:4
 * chroma, planar, semi-planar (NV12, P010 / P016) or packed (YUYV, UYVY).  Luma sample (r, c) of
 * frame f is the sample at byte y + f * y_frame_stride + r * y_pitch + c * luma_step * sample_bytes;
 * chroma sample (r, c) is at u + f * u_frame_stride + r * u_pitch + c * chroma_step * sample_bytes
 * (v likewise), with chroma planes of ceil(H / 2^chroma_shift_y) x ceil(W / 2^chroma_shift_x)
 * samples.  Each plane pointer gives its first sample, so interleaved layouts are three pointers
 * into one buffer: NV12 / P010 (chroma_step 2, v = u + sample_bytes), YUYV (luma_step 2,
 * chroma_step 4, u = y + 1, v = y + 3), UYVY (u = y - 1, v = y + 1).  Strides and pitches are in
 * bytes; 16-bit samples are little-endian and need 2-byte aligned planes, pitches and strides.
 *
 * Conversion contract: pixel (r, c) of the full frame uses chroma sample
 * (r >> chroma_shift_y, c >> chroma_shift_x) (nearest, absolute coordinates).  Each sample s is
 * first normalised to 16 bits: 8-bit v16 = s << 8; MSB-aligned 16-bit (P010 / P016) v16 = s;
 * LSB-aligned (yuv420p10le) v16 = (s & (2^bits - 1)) << (16 - bits).  With C = Y16 - 4096,
 * k = 298 (limited range) or C = Y16, k = 256 (full range), D = U16 - 32768, E = V16 - 32768:
 *   R = (k*C + cr*E + 32768) >> 16, G = (k*C - gu*D - gv*E + 32768) >> 16,
 *   B = (k*C + bu*D + 32768) >> 16
 * (int32 arithmetic shift, then clamped to [0, 255]) with the (cr, gu, gv, bu) table of
 * tapir_yuv420_frames plus BT.2020 (non-constant luminance; round(256 x coefficient) like the
 * other rows): limited (430, 48, 167, 548), full (377, 42, 146, 482).  For 8-bit samples this is
 * the tapir_yuv420_frames contract exactly ((256 S + 32768) >> 16 == (S + 128) >> 8), so 16-bit
 * samples holding 8-bit values in their high byte convert to the bytes of the 8-bit frame.  As
 * there, everything after the conversion is the uint8 RGB path. */
typedef struct tapir_yuv_frames {
  const void* y;
  const void* u;
  const void* v;
  int64_t y_frame_stride, u_frame_stride, v_frame_stride;
  int64_t y_pitch, u_pitch, v_pitch;
  int32_t H, W;                  /* full frame (luma samples) */
  int32_t y0, x0, h, w;          /* crop window inside the frame */
  int32_t matrix;                /* 601, 709 or 2020 */
  int32_t full_range;            /* 0: limited (16-235 luma at 8 bits), 1: full */
  int32_t sample_bytes;          /* 1 or 2 */
  int32_t bits;                  /* 8 (sample_bytes 1) or 8..16 (sample_bytes 2) */
  int32_t lsb_aligned;           /* 16-bit samples: 0 MSB-aligned (P010), 1 LSB-aligned */
  int32_t luma_step;             /* samples between luma samples of a row: 1 planar, 2 packed */
  int32_t chroma_step;           /* >= 1: 1 planar, 2 semi-planar, 4 packed 4:2:2 */
  int32_t chroma_shift_x;        /* 0 or 1: 1 for 4:2:0 and 4:2:2, 0 for 4:4:4 */
  int32_t chroma_shift_y;        /* 0 or 1: 1 for 4:2:0, 0 for 4:2:2 and 4:4:4 */
  int32_t reserved;
} tapir_yuv_frames;

/* tapir_yuv420_to_rgb, tapir_ingest_frames_yuv420 and tapir_backbone_forward_yuv420 for any
 * tapir_yuv_frames layout (the 4:2:0 calls run the same kernels).  Every descriptor field is
 * checked before any launch; a bad one returns 1. */
int tapir_yuv_to_rgb(const tapir_yuv_frames* src, int32_t frames, uint8_t* dst, void* stream);
int tapir_ingest_frames_yuv(const tapir_yuv_frames* src, int32_t frames, float* dst, int32_t oH,
                            int32_t oW, void* stream);

/* One source frame of tapir_ingest_frames_multi: its own format, size, row pitch and crop window.
 * TAPIR_INGEST_U8: pixel (r, c) of the frame is src[r * pitch + c * 3 ...] (bytes; pitch >= 3 W)
 * and the window (y0, x0, h, w) lies inside the H x W frame.  TAPIR_INGEST_YUV420 reads frame 0 of
 * `yuv` inside its own window (src, pitch, H, W and the window fields are then not read).
 * TAPIR_INGEST_YUV reads frame 0 of the tapir_yuv_frames `src` points to, inside its own window;
 * pitch, H, W and the window fields must then be 0.  fp32
 * frames are not covered: the blend of tapir_bilinear_resize rounds differently (its taps are
 * contracted into FMAs in another order), so they keep one tapir_bilinear_resize call each. */
#define TAPIR_INGEST_U8 1     /* uint8 RGB [0, 255] (tapir_ingest_frames' input) */
#define TAPIR_INGEST_YUV420 2 /* 8-bit YUV 4:2:0 (tapir_ingest_frames_yuv420's input) */
#define TAPIR_INGEST_YUV 3    /* any tapir_yuv_frames layout (tapir_ingest_frames_yuv's input) */
typedef struct tapir_ingest_desc {
  const void* src;
  int64_t pitch;
  int32_t format;
  int32_t H, W;
  int32_t y0, x0, h, w;
  int32_t reserved;
  tapir_yuv420_frames yuv;
} tapir_ingest_desc;

/* Frames of different sizes and formats -> dst [frames][oH][oW][3] float in [-1,1], frame i from
 * descs[i] (a host array).  Output frame i equals, bit for bit, what the one-format call gives for
 * that frame alone: tapir_ingest_frames (uint8) or tapir_ingest_frames_yuv420 on its window.
 * One launch per TAPIR_INGEST_MAX_FRAMES frames.  Every descriptor is checked before any CUDA call:
 * a bad one returns 1. */
#define TAPIR_INGEST_MAX_FRAMES 64
int tapir_ingest_frames_multi(const tapir_ingest_desc* descs, int32_t frames, float* dst,
                              int32_t oH, int32_t oW, void* stream);

/* tapir_backbone_forward_ex on the crop window (h x w) of YUV 4:2:0 frames: the conversion and
 * the normalisation run inside the stem conv's loads; same launches as the uint8 reader. */
int tapir_backbone_forward_yuv420(const tapir_backbone_weights* w, const tapir_yuv420_frames* video,
                                  int32_t frames, float* lowres, float* hires, void* workspace,
                                  size_t workspace_bytes, void* hires_ready_event, void* stream);
int tapir_backbone_forward_yuv(const tapir_backbone_weights* w, const tapir_yuv_frames* video,
                               int32_t frames, float* lowres, float* hires, void* workspace,
                               size_t workspace_bytes, void* hires_ready_event, void* stream);

/* ---- SURVEY 8f row 2: output post-processing (the step after the path) ---------------- */
/* pytorch_live_demo.py:57-59 / utils/model_utils.py:376-389:
 * visible[i] = (1 - sigmoid(occ[i])) * (1 - sigmoid(expd[i])) > 0.5 */
int tapir_postprocess_occlusions(const float* occ, const float* expd, int64_t n, uint8_t* visible,
                                 void* stream);

/* tapvid/evaluation_datasets.py:48-192 compute_tapvid_metrics, as exact integer counters per
 * track; the host forms the ratios from their sums.  counts [B][N][TAPIR_TAPVID_COUNTERS]:
 * [0] evaluated frames, [1] occlusion prediction correct, [2] ground-truth visible,
 * [3+i] within 2^i px and visible, [8+i] true positives, [13+i] false positives (i = 0..4). */
#define TAPIR_TAPVID_COUNTERS 18
typedef struct {
  const float* query_points;    /* [B][N][3]  (t, y, x) */
  const uint8_t* gt_occluded;   /* [B][N][T]  bool */
  const float* gt_tracks;       /* [B][N][T][2] (x, y) */
  const uint8_t* pred_occluded; /* [B][N][T] bool, or NULL to threshold the two logit arrays */
  const float* pred_occ_logits; /* [B][N][T] (used when pred_occluded is NULL) */
  const float* pred_expd_logits;
  const float* pred_tracks;     /* [B][N][T][2] */
  int32_t B, N, T;
  int32_t query_mode;           /* 0 = 'first', 1 = 'strided' */
  int32_t* counts;
} tapir_tapvid_args;
int tapir_tapvid_counts(const tapir_tapvid_args* args, void* stream);

/* tapnextpp/metrics/aj_rd.py compute_raw_redetection_stats: the eligible reappearance events of
 * every track (b, n) and their AJ_RD values, bit for bit.  A reappearance is a frame t >= 1 with
 * gt_visible[t] && !gt_visible[t-1]; its duration is the length of the invisible run ending at
 * t - 1 (t itself if the track is invisible from frame 0).  An event is eligible when its duration
 * is strictly greater than every earlier event's of the track.  For threshold D, over frames
 * [t, T): within = sqrt_rn(fma(dy, dy, dx * dx)) <= D (float32, a NaN distance is not within),
 * TP = sum(within && gt && pred), FP = sum(pred && (!gt || !within)), value = float(TP) /
 * float(sum(gt) + FP) (IEEE float32; 0 / 0 is NaN).
 *
 * A track has at most K(T) eligible events, K(T) the largest k with k (k + 3) / 2 <= T (their
 * durations are at least 1 .. k, each followed by a visible frame); tapir_redetection_max_events
 * (host only) returns K(T) (0 for T < 1).  Track i = b N + n writes its events, in t order, to
 * slots i K(T) .. i K(T) + event_count[i] - 1 of event_t, event_duration and event_values
 * [slot][num_thresholds]; the other slots are not written.  event_* need capacity >= B N K(T)
 * slots (they may be NULL when K(T) = 0).  No allocation, no host copy, no host sync: graph-
 * capturable.  A bad argument returns 1 before any CUDA call. */
#define TAPIR_REDETECTION_MAX_THRESHOLDS 16
typedef struct {
  const uint8_t* gt_visible;    /* [B][N][T] bool */
  const uint8_t* pred_visible;  /* [B][N][T] bool, or NULL to threshold the two logit arrays as
                                   tapir_tapvid_counts does */
  const float* pred_occ_logits; /* [B][N][T] (used when pred_visible is NULL) */
  const float* pred_expd_logits;
  const float* pred_tracks;     /* [B][N][T][2] (x, y) */
  const float* gt_tracks;       /* [B][N][T][2] */
  float thresholds[TAPIR_REDETECTION_MAX_THRESHOLDS]; /* distance thresholds D, float32 */
  int32_t num_thresholds;       /* 1 .. TAPIR_REDETECTION_MAX_THRESHOLDS */
  int32_t B, N, T;
  int64_t capacity;             /* slots of event_t / event_duration / event_values */
  int32_t* event_t;             /* [capacity] reappearance frame */
  int32_t* event_duration;      /* [capacity] */
  float* event_values;          /* [capacity][num_thresholds] */
  int32_t* event_count;         /* [B][N] */
} tapir_redetection_args;
int32_t tapir_redetection_max_events(int32_t T);
int tapir_redetection_events(const tapir_redetection_args* args, void* stream);

/* ---- f5: visualisation (the step after the path) ------------------------------------- */
/* tapnet/utils/viz_utils.py:47-124 paint_point_track, bit for bit: frames [T][H][W][3] uint8 ->
 * out (same shape, must not overlap frames) with a dot of radius round(min(H, W) * 0.015) at
 * every visible point, painted in index order.  tracks [N][T][2] (x, y) float (tracks_fp64 = 0)
 * or double (1); the + 0.5 to the dot centre is taken in that dtype.  visibles [N][T] uint8
 * (non-zero paints), colors [N][3] uint8.  Points with a NaN coordinate are skipped (undefined in
 * the reference).  N = 0 copies the frames.  Workspace: tapir_paint_point_track_workspace_bytes
 * (T, N) bytes, 16-byte aligned (NULL when N = 0).  Two launches; stream-ordered, no host sync.
 * A bad argument (negative size, NULL pointer, small workspace, out overlapping frames) returns
 * 1 before any CUDA call. */
size_t tapir_paint_point_track_workspace_bytes(int32_t frames, int32_t points);
int tapir_paint_point_track(const uint8_t* frames, int32_t T, int32_t H, int32_t W,
                            const void* tracks, int32_t tracks_fp64, const uint8_t* visibles,
                            int32_t N, const uint8_t* colors, uint8_t* out, void* workspace,
                            size_t workspace_bytes, void* stream);

/* ---- f8: camera homographies from point tracks (the step after the path) --------------- */
/* viz_utils.py:301-648 get_homographies_wrt_frame in float64: one homography per frame that maps
 * background points into the reference frame, each track's squared distance to its canonical
 * point per frame, and the canonical points.  tracks [N][T][2] (x, y pixels) float
 * (tracks_fp64 = 0) or double (1); occluded [N][T] uint8 (non-zero = occluded).  stop_thresholds
 * is a device copy of tapir_ransac_stop_thresholds(N, targ_inlier_frac).  Outputs: homogs
 * [T][3][3], err [N][T], canonical [N][2] (double); ransac_stats [T][2] int32 (hypotheses
 * evaluated, best inlier count per frame of the initial sweep; 0 / 0 for the reference frame and
 * frames with <= 4 usable points) or NULL.  RANSAC draws come from a fixed SplitMix64 stream, so
 * the result is a function of the inputs.  Workspace: tapir_homographies_workspace_bytes(T, N),
 * 256-byte aligned.  Launches per frame step: 4 in the initial sweep, 2 per refinement step (3 for
 * the reference frame of a pass before the last), plus 2; no allocation, no host sync.  Every
 * argument is checked first; a bad one returns 1 before any CUDA call. */
typedef struct {
  const void* tracks;            /* [N][T][2] */
  int32_t tracks_fp64;           /* 0: float, 1: double */
  int32_t N, T;
  int32_t reference_frame;       /* 0 .. T-1 */
  const uint8_t* occluded;       /* [N][T] */
  double width, height;          /* image size in pixels, > 0 */
  double thresh;                 /* outlier threshold in normalised coordinates, > 0 */
  double outlier_point_threshold;/* required inlier fraction of a canonical point, > 0 */
  int32_t num_refinement_passes; /* >= 0 */
  int32_t reserved;
  const double* stop_thresholds; /* [N] device */
  double* homogs;                /* [T][3][3] */
  double* err;                   /* [N][T] */
  double* canonical;             /* [N][2] */
  int32_t* ransac_stats;         /* [T][2] or NULL */
  void* workspace;
  size_t workspace_bytes;
} tapir_homography_args;
/* Host only: thr[it] = min(1 - (it + 1) / N, targ_inlier_frac * pow(0.99, it)) * N for it in
 * 0 .. N-1 into the host array out (libm pow).  RANSAC stops after hypothesis k once its best
 * count is >= thr[k + 1].  Bad arguments return 1. */
int tapir_ransac_stop_thresholds(int32_t N, double targ_inlier_frac, double* out);
/* 0 for T < 1 or N < 1. */
size_t tapir_homographies_workspace_bytes(int32_t T, int32_t N);
int tapir_homographies_wrt_frame(const tapir_homography_args* args, void* stream);

/* ---- f6: evaluation (the step before the path) -------------------------------------- */
/* tapvid/evaluation_datasets.py:41-45 resize_video on uint8 RGB frames, bit for bit as PIL's
 * Image.resize(..., LANCZOS) (what mediapy.resize_video runs per uint8 frame).  Per axis
 * (in -> out): scale = in / out, fs = max(scale, 1), ksize = 2 ceil(3 fs) + 1; output o reads
 * inputs xmin .. xmin + n - 1 with taps lanczos((i + xmin - c + 0.5) * (1 / fs)), c = (o + 0.5) scale,
 * normalised in double and rounded half away from zero to 22 fraction bits; a pass is
 * clamp((2^21 + sum src * tap) >> 22, 0, 255) in int32.
 *
 * tapir_lanczos_weights is host only (no GPU): for sizes in 1..TAPIR_MAX_RESIZE_SIDE it returns
 * ksize and, unless they are NULL, fills the host arrays bounds [out_size][2] (xmin, n) and
 * taps [out_size][ksize] int32; bad sizes return -1 with tapir_last_error() set. */
#define TAPIR_MAX_RESIZE_SIDE 65535
int32_t tapir_lanczos_weights(int32_t in_size, int32_t out_size, int32_t* bounds, int32_t* taps);
/* Workspace of tapir_resize_lanczos_u8: the uint8 intermediate of the rows the vertical pass reads
 * (0 unless both W != w and H != h); 0 for bad sizes. */
size_t tapir_resize_lanczos_u8_workspace_bytes(int32_t frames, int32_t H, int32_t W, int32_t h,
                                               int32_t w);
/* src [frames][H][W][3] uint8 -> dst [frames][h][w][3] uint8: a horizontal pass (if W != w) into
 * a uint8 intermediate, then a vertical pass (if H != h); equal sizes copy.  x_* are the device
 * copies of tapir_lanczos_weights(W, w) (with its ksize), y_* of tapir_lanczos_weights(H, h); the
 * tables of an axis that keeps its size are not read and may be NULL.  Workspace 16-byte aligned,
 * at least tapir_resize_lanczos_u8_workspace_bytes (NULL when that is 0).  No allocation, no
 * host <-> device copy, no host sync: graph-capturable.  A bad argument (size, NULL pointer, table
 * size, workspace size or alignment, dst or workspace overlapping src) returns 1 before any CUDA
 * call. */
int tapir_resize_lanczos_u8(const uint8_t* src, uint8_t* dst, int32_t frames, int32_t H, int32_t W,
                            int32_t h, int32_t w, const int32_t* x_bounds, const int32_t* x_taps,
                            int32_t x_ksize, const int32_t* y_bounds, const int32_t* y_taps,
                            int32_t y_ksize, void* workspace, size_t workspace_bytes, void* stream);

/* ---- a4: tapir_model.py:217-291 + utils.py:45-73 (trilinear, border clamp) ---------- */
/* query_tyx [N][3] in video coordinates (vT,vH,vW) -> out [N][C] */
int tapir_sample_query_features(const float* grid, int32_t T, int32_t gh, int32_t gw, int32_t C,
                                const float* query_tyx, int32_t N, int32_t vT, int32_t vH,
                                int32_t vW, float* out, void* stream);
/* The same sampling from a grid [T][gh][gw][C] that holds only some frames of a vT-frame clip:
 * frame_slot (int32 [vT]) maps each clip frame to its slot in the grid, or -1 for a frame the grid
 * does not hold.  The clip's vT normalises the time axis, so a query's features are bit for bit
 * those sampled from the whole clip's grid whenever every tap of nonzero weight lands on a held
 * frame; a query with such a tap on an absent frame gets a NaN row instead (the grid is never read
 * outside its T slots).  frame_slot == NULL is tapir_sample_query_features: same launch, same
 * results.  Every argument is checked first (sizes, NULL pointers, 4-byte alignment, out
 * overlapping an input); a bad one returns 1 before any CUDA call. */
int tapir_sample_query_features_ex(const float* grid, int32_t T, int32_t gh, int32_t gw, int32_t C,
                                   const float* query_tyx, int32_t N, int32_t vT, int32_t vH,
                                   int32_t vW, const int32_t* frame_slot, float* out, void* stream);

/* ---- a6: tapir_model.py:687-761 + utils.py:116-193 --------------------------------- */
size_t tapir_cost_volume_workspace_bytes(int32_t N, int32_t T, int32_t gh, int32_t gw, int32_t C);
/* qfeat [N][C], grid [T][gh][gw][C] (gh=gw=32 supported), query_tyx [N][3] in
 * initial_resolution pixel coordinates or NULL.  Outputs: points [N][T][2] (x,y in
 * initial_resolution pixels), occ/expd logits [N][T], argmax [N][T] flat cell index
 * (nullable). */
int tapir_cost_volume_tracks(const tapir_head_weights* w, const float* qfeat, const float* grid,
                             int32_t N, int32_t T, int32_t gh, int32_t gw, int32_t C,
                             const float* query_tyx, float softmax_temperature, int32_t init_h,
                             int32_t init_w, float* points, float* occ, float* expd,
                             int32_t* argmax, void* workspace, size_t workspace_bytes,
                             void* stream);

/* The same for B clips in one launch sequence: qfeat [B][N][C], grid [B][T][gh][gw][C],
 * query_tyx [B][N][3] or NULL; outputs as above over the flattened query b*N + n.  One batched
 * GEMM and one head launch; clip b's results equal those of a tapir_cost_volume_tracks call on
 * clip b alone, bit for bit.  B*N <= 65535 for the 32 x 32 map.  B = 1 is
 * tapir_cost_volume_tracks. */
size_t tapir_cost_volume_batched_workspace_bytes(int32_t B, int32_t N, int32_t T, int32_t gh,
                                                 int32_t gw, int32_t C);
int tapir_cost_volume_tracks_batched(const tapir_head_weights* w, const float* qfeat,
                                     const float* grid, int32_t B, int32_t N, int32_t T, int32_t gh,
                                     int32_t gw, int32_t C, const float* query_tyx,
                                     float softmax_temperature, int32_t init_h, int32_t init_w,
                                     float* points, float* occ, float* expd, int32_t* argmax,
                                     void* workspace, size_t workspace_bytes, void* stream);

/* The same for B clips with their own query counts: points_per_clip is a HOST array of B counts
 * N_b >= 1 (1 <= B <= TAPIR_MAX_RAGGED_CLIPS), qfeat [sum N_b][C] and query_tyx [sum N_b][3] (or
 * NULL) hold the clips' queries one clip after the other, grid is [B][T][gh][gw][C]; outputs run
 * over the flattened query as above.  One grouped GEMM and one head launch, no host-to-device
 * copy (the call may be captured in a CUDA graph); clip b's results equal those of a
 * tapir_cost_volume_tracks call on clip b alone, bit for bit.  sum N_b <= 65535 for the 32 x 32
 * map.  Every argument is checked first; a bad one returns 1 before any CUDA call.  The workspace
 * depends on the clip count and the total query count only. */
size_t tapir_cost_volume_ragged_workspace_bytes(int32_t B, int32_t total_points, int32_t T,
                                                int32_t gh, int32_t gw, int32_t C);
int tapir_cost_volume_tracks_ragged(const tapir_head_weights* w, const float* qfeat,
                                    const float* grid, int32_t B, const int32_t* points_per_clip,
                                    int32_t T, int32_t gh, int32_t gw, int32_t C,
                                    const float* query_tyx, float softmax_temperature,
                                    int32_t init_h, int32_t init_w, float* points, float* occ,
                                    float* expd, int32_t* argmax, void* workspace,
                                    size_t workspace_bytes, void* stream);

/* ---- point edits of a one-frame step (pytorch_live_demo.py:180-206 re-targets a point) ----
 * tapir_sample_query_rows applies a request table to a group of `clips` one-frame clips whose
 * queries are packed along one point axis of `rows` rows.  Request r < *count (count is read on
 * the device, so one captured launch serves any number of requests; at most `rows` are read):
 *  - samples, for every grid i, grids[i].grid of clip `clip` at (t, y, x) into row `row` of
 *    grids[i].out, exactly as tapir_sample_query_features on that clip alone with vT = T = 1;
 *    the clip's video size is video_hw[clip] (a device int32 table [clips][2]) or, when video_hw
 *    is NULL, video_h x video_w;
 *  - zeroes row `row` of every causal-state tensor: `state` is a device table of num_state
 *    pointers, entry 2k a [rows][2][512] tensor (ctx1) and entry 2k + 1 a [rows][2][2048] tensor
 *    (ctx2), each 16-byte aligned.
 * A request whose row or clip is out of range is skipped.  Rows without a request are not
 * touched.  `grids` is a HOST array; nothing is allocated or copied, so the call may be captured
 * in a CUDA graph.  Every argument is checked first; a bad one returns 1 before any CUDA call. */
#define TAPIR_MAX_QUERY_GRIDS 16 /* a lowres and a hires grid per resolution level */
typedef struct tapir_query_grid {
  const float* grid;   /* [clips][h][w][C]: clip c's one-frame grid at grid + c * clip_stride */
  int64_t clip_stride; /* in floats, >= h * w * C */
  float* out;          /* [rows][C] packed query features */
  int32_t h, w, C, reserved;
} tapir_query_grid;
typedef struct tapir_query_request {
  int32_t row, clip; /* the point's row in the packed point axis, its clip in the group */
  float t, y, x;     /* the query point in the clip's video pixels */
} tapir_query_request;
int tapir_sample_query_rows(const tapir_query_grid* grids, int32_t num_grids, int32_t clips,
                            int32_t rows, int32_t video_h, int32_t video_w, const int32_t* video_hw,
                            const int32_t* count, const tapir_query_request* requests,
                            float* const* state, int32_t num_state, void* stream);

/* ---- a9: tapir_model.py:519-527 avg_pool3d (2,2,1) ---------------------------------- */
int tapir_pool_pyramid(const float* grid, int32_t T, int32_t h, int32_t w, int32_t C, float* out,
                       void* stream);

/* ---- a7 / a8 ------------------------------------------------------------------------ */
int tapir_local_corr(const tapir_corr_args* args, void* stream);
/* `batch` clips in one launch: args->num_points = queries per clip; every level grid is
 * [batch][T][h][w][C]; pos / occ / expd / features / output rows run over the flattened query
 * b*num_points + n.  Equal to one tapir_local_corr call per clip, bit for bit. */
int tapir_local_corr_batched(const tapir_corr_args* args, int32_t batch, void* stream);
/* `batch` clips with their own query counts: args->num_points = the queries of all clips,
 * query_clip a device int32 table [num_points] giving each flattened query's clip (in
 * 0..batch-1), whose level grids [batch][T][h][w][C] it reads.  Equal to one tapir_local_corr
 * call per clip, bit for bit.  Every argument is checked first; a bad one returns 1. */
int tapir_local_corr_ragged(const tapir_corr_args* args, int32_t batch, const int32_t* query_clip,
                            void* stream);
size_t tapir_mixer_workspace_bytes(int64_t rows, int32_t planes);
int tapir_mixer_forward(const tapir_mixer_weights* w, const tapir_mixer_io* io, void* workspace,
                        size_t workspace_bytes, void* stream);
/* The depthwise half of one mixer block, the kernel tapir_mixer_forward runs between its GEMMs
 * (nets.py:143-181 up to the channel MLP): x [n][T][512] fp32 -> z = x + group sum of the two
 * depthwise convs [n][T][512] fp32, and LayerNorm_1(z) * ln1_w as `planes` bf16 planes
 * [planes][n*T][512] at `plane_stride` elements.  causal != 0: causal convs, with the optional
 * context of tapir_mixer_io (ctx1 [n][2][512], ctx2 [n][2][2048]; NULL = zero context / not
 * requested); a non-causal call takes no context pointers.  A context output may be its input
 * buffer only at T = 1.  Every argument is checked before any CUDA call (NULLs, n in 1..65535,
 * T >= 1, planes 1..3, overlapping planes, 16-byte alignment of x, z, the contexts and the
 * LayerNorm weights): a bad one returns 1. */
int tapir_mixer_dw(const tapir_mixer_block* blk, const float* x, int32_t n, int32_t T, int32_t causal,
                   const float* ctx1_in, const float* ctx2_in, float* ctx1_out, float* ctx2_out, float* z,
                   void* planes_out, int64_t plane_stride, int32_t planes, void* stream);
int tapir_refine_update(const tapir_update_args* args, void* stream);
/* tapir_refine_update over a batch of clips of different video sizes: video_hw is a device int32
 * table [clips][2] of (video_h, video_w), and row r (= query * num_frames + frame) belongs to
 * clip r / rows_per_clip; tracks_out of that row is scaled to its clip's size (args->video_h /
 * video_w are not read).  Each clip's rows equal a tapir_refine_update call with its size, bit for
 * bit.  video_hw = NULL is tapir_refine_update. */
int tapir_refine_update_ex(const tapir_update_args* args, const int32_t* video_hw,
                           int32_t rows_per_clip, void* stream);
/* tapir_refine_update over clips with their own query counts and video sizes: row r = q *
 * num_frames + t takes its clip's (video_h, video_w) from video_hw[query_clip[q]], where
 * query_clip is a device int32 table [num_points] and video_hw a device int32 table [clips][2].
 * Each clip's rows equal a tapir_refine_update call with its size, bit for bit.  Every argument is
 * checked first; a bad one returns 1. */
int tapir_refine_update_ragged(const tapir_update_args* args, const int32_t* video_hw,
                               const int32_t* query_clip, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* TAPIR_B200_H_ */
