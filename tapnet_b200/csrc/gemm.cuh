// Split-bf16 GEMM / implicit-GEMM 3x3 convolution: host-side description shared by the
// wgmma kernel (gemm_tc.cu) and the SIMT verification kernel (gemm_simt.cu).
//
//   D[m, n] = sum_{i + j < P} sum_k A_i[m, k] * B_j[n, k]        (fp32 accumulation)
//   v = D + bias[n];  v = act ? gelu_tanh(v) : v;  v += residual[m, n]
//   out_f32[m, n] = v   and / or   out_planes[q][m, n] = q-th bf16 term of v
//
// A_i, B_j are the bf16 "planes" of an fp32 tensor (x ~= p0 + p1 (+ p2), see
// split_bf16 in common.cuh).  P=1 is plain bf16, P=2 (3 MMAs) carries ~16 mantissa bits,
// P=3 (6 MMAs) is fp32-equivalent.  The reference computes every one of these contractions
// in fp32 (tapir_model.py:665,720; nets.py convs/linears), and its parity budget (1e-3 px,
// 1e-4 logits) cannot be met by single-pass bf16 (tests/test_precision_policy.py).
#pragma once
#include "../../include/tapir_b200.h"
#include "common.cuh"

namespace tapir {

enum GemmMode : int { kGemmPlain = 0, kGemmConv3x3 = 1 };

// Most problems of one grouped GEMM (GemmArgs::groups); TAPIR_MAX_RAGGED_CLIPS in the C ABI.
constexpr int kGemmMaxGroups = TAPIR_MAX_RAGGED_CLIPS;

struct GemmArgs {
  int mode = kGemmPlain;
  int planes = 2;  // P
  int M = 0, N = 0, K = 0;  // K: contraction length, multiple of 64 (conv: 9*C)
  // A: plain -> [P][M][lda] bf16; conv -> [P][frames][H][W][C] bf16 (NHWC), M = frames*H*W
  const __nv_bfloat16* a = nullptr;
  int lda = 0;
  long long a_plane_stride = 0;  // elements between planes
  int frames = 0, H = 0, W = 0, C = 0;
  // B: [P][N][ldb] bf16 (row n holds the K weights of output channel n; conv K order is
  // (ky, kx, c))
  const __nv_bfloat16* b = nullptr;
  int ldb = 0;
  long long b_plane_stride = 0;
  // epilogue
  const float* bias = nullptr;      // [N]
  const float* residual = nullptr;  // [M][ldr]
  int ldr = 0;
  int act = 0;                      // 1 = tanh-GELU
  float* out_f32 = nullptr;         // [M][ldo]
  int ldo = 0;
  __nv_bfloat16* out_planes = nullptr;  // [out_P][M][ldp]
  int ldp = 0;
  long long out_plane_stride = 0;
  int out_P = 0;
  double* stats = nullptr;  // optional fused per-(frame, column) sum / sum-of-squares (fp64)
  int rows_per_frame = 0;   // plain mode: rows per frame (multiple of 128); conv: implied
  float* splitk_ws = nullptr;  // optional scratch enabling split-K for under-filled problems
  size_t splitk_ws_bytes = 0;
  // Callers set this for single-frame (streaming) steps only: a split GEMM sums K in a different
  // order, so allowing it by problem size alone would make an offline result depend on how its
  // rows were chunked or sharded (measured: 1.5e-5 on occlusion logits).
  bool allow_splitk = false;
  // Batched plain GEMM: `batch` independent problems of M x N, batch b reading A rows
  // [b * a_batch_rows, + M) and B rows [b * b_batch_rows, + N) of the flattened operand planes and
  // writing out_f32 + b * out_batch_stride.  An m-tile never crosses a batch.  batch > 1 supports
  // the fp32 output, bias and GELU only, and never splits K.
  int batch = 1;
  long long a_batch_rows = 0;      // 0 = M
  long long b_batch_rows = 0;      // 0 = N
  long long out_batch_stride = 0;  // elements; 0 = M * ldo
  // Grouped plain GEMM (groups > 0, batch 1): problem g owns A rows and output rows
  // [group_row0[g], group_row0[g + 1]) and B rows [g * b_batch_rows, + N); M is the rows of all
  // groups (group_row0[groups]).  An m-tile never crosses a group; rows of a group's last tile
  // past its end are loaded but never stored.  The same epilogue limits as batch > 1, and K is
  // never split.  The table travels in the kernel parameters, so a call needs no device copy.
  int groups = 0;
  int group_row0[kGemmMaxGroups + 1] = {};
  int k_logical = 0;       // un-padded K for FLOP accounting (0 = K)
  const char* tag = nullptr;  // profiling class name
};

// A GEMM with weight `l` as its B operand and bias; the caller sets A, M and the outputs.
inline GemmArgs gemm_args(const tapir_linear& l) {
  GemmArgs g;
  g.planes = l.planes;
  g.N = l.N;
  g.K = l.K;
  g.b = static_cast<const __nv_bfloat16*>(l.w);
  g.ldb = l.K;
  g.b_plane_stride = (long long)l.N * l.K;
  g.bias = l.bias;
  g.k_logical = l.k_logical;
  return g;
}

// Overrides of the GEMM dispatcher's choices, from environment variables.  read_gemm_switches reads
// all four on every GEMM call, whether the call uses them or not.  Unset leaves the choice to the
// dispatcher; any other value than those listed, the empty string included, fails the call with
// kBadArgument before anything is launched.
//   TAPIR_B200_GEMM           tc | simt        simt: gemm() runs the SIMT cross-check kernel
//   TAPIR_B200_BLOCK_N        64 | 128         the wgmma kernel's tile width
//   TAPIR_B200_GEMM_SCHEDULE  coop | pingpong  the wgmma schedule, wherever both are legal
//   TAPIR_B200_CONV_HALO      0 | 1            0: C = 64 3x3 convolutions take the generic path
struct GemmSwitches {
  bool simt = false;
  int block_n = 0;   // 0: not set
  int schedule = 0;  // 0: not set, 1: coop, 2: pingpong
  bool halo = true;
};
int read_gemm_switches(GemmSwitches* sw);

int validate_gemm_args(const GemmArgs& g);
// wgmma + TMA implementation (the product path).
int gemm_tc(const GemmArgs& g, const GemmSwitches& sw, cudaStream_t stream);
// Straightforward SIMT implementation of the same arithmetic (verification / bring-up).
int gemm_simt(const GemmArgs& g, cudaStream_t stream);
// gemm_simt under TAPIR_B200_GEMM=simt, else gemm_tc.
int gemm(const GemmArgs& g, cudaStream_t stream);

}  // namespace tapir
