// wgmma / TMA split-bf16 GEMM and implicit-GEMM 3x3 convolution for sm_90a.
//
// One persistent CTA per SM, three warpgroups:
//   warpgroup 0 (one lane)  TMA producer: cp.async.bulk.tensor tiles of A and B planes into a
//                           multi-stage shared-memory ring (128B-swizzled, K-major)
//   warpgroups 1, 2         consumers: issue wgmma.m64nBLOCK_Nk16 (bf16 operands from shared
//                           memory, fp32 accumulators in registers) and then run the epilogue
//                           from their registers: bias / tanh-GELU / residual, fp32 and/or
//                           bf16-plane stores (whole ping-pong GEMM tiles of GELU + two planes:
//                           through shared memory and TMA stores).  Cooperative schedule: each
//                           owns 64 rows of every 128-row tile.  Ping-pong schedule: each owns
//                           whole tiles, alternately.
// full/empty mbarriers between producer and consumers; the producer runs ahead into the next
// tile while the consumers are in the epilogue of the current one.
//
// The four kernels are one body, wgmma_kernel<operand source, schedule>: gemm_tc_kernel and
// gemm_tc_pingpong_kernel over the stage ring (Ring), conv3x3_halo_kernel and
// conv3x3_halo_pingpong_kernel over the halo patch ring and its B ring (HaloRing).
//
// A operand, plain mode: 3-D tensor map {K, M, plane}, box {64, 128, 1}.
// A operand, conv mode : 5-D tensor map {C, W, H, frame, plane} over the NHWC activation,
//   box {64, tileW, tileH, 1, 1}; the 3x3 taps are shifted box origins, and TMA's
//   out-of-bounds zero fill implements the zero padding (nets.py:296-303,40-53 padding=1).
// B operand: 3-D tensor map {K, N, plane}, box {64, BLOCK_N, 1}.
//
// Every output element accumulates its K terms in the same order (k-block, then plane pair
// (i, j), then 16-wide k step) whatever the tile shape, so results do not depend on BLOCK_N.
#include <cuda.h>

#include <cstdlib>

#include "gemm.cuh"
#include "ptx.cuh"

namespace tapir {

namespace {

constexpr int kBlockM = 128;
constexpr int kBlockK = 64;  // 64 bf16 = 128 B = one swizzle row
constexpr int kMmaK = 16;
constexpr int kConsumers = 2;             // warpgroups, 64 rows each
constexpr int kThreads = 128 * (1 + kConsumers);
constexpr int kConsumerArrivals = 4 * kConsumers;  // one arrive per consumer warp
constexpr int kSmemLimit = 227 * 1024;
constexpr int kBarrierBytes = 256;

struct TcParams {
  CUtensorMap tmA;
  CUtensorMap tmB;
  CUtensorMap tmPatch;  // halo convolution: one patch row {64 ch, 10 px} per load
  CUtensorMap tmPlanes;  // ping-pong, plane_tma: output planes {N, M, 2}, stored in boxes {64, 64, 1}
  int plane_tma;         // whole ping-pong tiles write GELU + two planes through epilogue_planes_tma
  int frames;
  int M, N;
  int num_k_blocks;
  int num_m_tiles, num_n_tiles;
  int mode;
  int H, W, cblocks, tileW, tileH, tiles_x, tiles_y;
  const float* bias;
  const float* residual;
  int ldr;
  int act;
  float* out_f32;
  int ldo;
  __nv_bfloat16* out_planes;
  int ldp;
  long long out_plane_stride;
  int out_P;
  double* stats;        // optional [frames][N][2] column (sum, sum of squares) accumulators
  int rows_per_frame;   // rows of one frame (plain mode; conv tiles never straddle frames)
  int split_k;          // >1: K is split over `split_k` work items; raw fp32 partials go to out_f32
  long long split_stride;  // elements between partial buffers (M * ldo)
  int m_tiles_per_batch;   // batched plain GEMM: m-tiles of one batch (= num_m_tiles when batch 1)
  long long a_batch_rows, b_batch_rows, out_batch_stride;
  int groups;  // grouped plain GEMM (GemmArgs::groups): group g's first row and first m-tile
  int group_row0[kGemmMaxGroups + 1], group_tile0[kGemmMaxGroups + 1];
  int* err;
};

// Ping-pong output staging (epilogue_planes_tma): per consumer warpgroup one 64 x 64 bf16 box
// buffer per output plane.
constexpr int kPlaneBoxBytes = 64 * 128;
constexpr int kPlaneStagingBytes = kConsumers * 2 * kPlaneBoxBytes;

// Shared memory: the stage ring, STAGING bytes after it, then the barriers.
template <int BLOCK_N, int P, int STAGING = 0>
struct TcCfg {
  static constexpr int kABytes = kBlockM * kBlockK * 2;
  static constexpr int kBBytes = BLOCK_N * kBlockK * 2;
  static constexpr int kStageBytes = P * (kABytes + kBBytes);
  static constexpr int kAvail = kSmemLimit - 1024 - STAGING - kBarrierBytes;
  static constexpr int kStagesRaw = kAvail / kStageBytes;
  static constexpr int kStages = kStagesRaw > 6 ? 6 : kStagesRaw;
  static constexpr int kSmemBytes = 1024 + kStages * kStageBytes + STAGING + kBarrierBytes;
  static_assert(kStages >= 2, "tile does not fit in shared memory");
  static_assert(kStages * 2 <= kBarrierBytes / 8, "barrier space");
};

template <int BLOCK_N>
__device__ __forceinline__ void wgmma_bf16(float (&d)[BLOCK_N / 2], uint64_t adesc, uint64_t bdesc,
                                           uint32_t accumulate) {
  if constexpr (BLOCK_N == 64) ptx::wgmma_m64n64k16(d, adesc, bdesc, accumulate);
  else ptx::wgmma_m64n128k16(d, adesc, bdesc, accumulate);
}

// Fused InstanceNorm statistics, per tile.  Each warp sums its 16 rows of a column in fp32 (a
// shuffle over the 8 lanes that hold the column) and puts the fp64 (sum, sum of squares) into its
// slot of the warpgroup's [4 warps][BLOCK_N][2] buffer in shared memory; under ping-pong the
// second 64-row half adds to the first's slots.  flush_stats then sums the four warps' slots in
// fp64 and issues one atomic per column and value: 2 BLOCK_N atomics per warpgroup and tile where
// every warp used to issue its own (8x fewer under ping-pong, 4x under the cooperative schedule).
template <int BLOCK_N>
constexpr int kStatsSlotBytes = 4 * BLOCK_N * 2 * 8;  // per consumer warpgroup

// Lanes 0-3 of a warp: its partials of columns cl, cl + 1 of the tile (st: sum cl, sum cl + 1,
// square cl, square cl + 1) into its slots `red`, added to what they hold when `add`.
__device__ __forceinline__ void put_stats(double* red, int cl, const float (&st)[4], bool add) {
  double2* r = reinterpret_cast<double2*>(red + 2 * cl);
  double2 a = make_double2(st[0], st[2]), b = make_double2(st[1], st[3]);
  if (add) {
    const double2 x = r[0], y = r[1];
    a.x += x.x; a.y += x.y; b.x += y.x; b.y += y.y;
  }
  r[0] = a;
  r[1] = b;
}

// Epilogue of a whole 64 x BLOCK_N accumulator whose rows and columns all exist, with the
// options fixed at compile time and vector accesses only: straight-line code without branches,
// so the compiler interleaves the independent column groups.  Each element goes through the
// same operations in the same order as in `epilogue` below, so the results are bit-identical.
template <int BLOCK_N, bool BIAS, bool GELU, bool RESID, bool F32, int PLANES, bool STATS>
__device__ __forceinline__ void epilogue_full(const TcParams& p, const float (&acc)[BLOCK_N / 2],
                                              const float* const (&res_row)[2], float* const (&out_row)[2],
                                              __nv_bfloat16* const (&pl_row)[2], int n0, int lane, double* red,
                                              bool add) {
#pragma unroll
  for (int j = 0; j < BLOCK_N / 8; ++j) {
    const int c = n0 + 8 * j + 2 * (lane & 3);
    float b0 = 0.f, b1 = 0.f;
    if constexpr (BIAS) { b0 = __ldg(p.bias + c); b1 = __ldg(p.bias + c + 1); }
    float st[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
      if constexpr (BIAS) { v0 += b0; v1 += b1; }
      if constexpr (GELU) { v0 = gelu_tanh(v0); v1 = gelu_tanh(v1); }
      if constexpr (RESID) {
        const float2 t = *reinterpret_cast<const float2*>(res_row[h] + c);
        v0 += t.x; v1 += t.y;
      }
      if constexpr (F32) *reinterpret_cast<float2*>(out_row[h] + c) = make_float2(v0, v1);
      if constexpr (STATS) { st[0] += v0; st[2] += v0 * v0; st[1] += v1; st[3] += v1 * v1; }
#pragma unroll
      for (int q = 0; q < PLANES; ++q)
        *reinterpret_cast<uint32_t*>(pl_row[h] + q * p.out_plane_stride + c) = bf16x2_split(v0, v1);
    }
    if constexpr (STATS) {
#pragma unroll
      for (int s = 4; s < 32; s <<= 1)
#pragma unroll
        for (int e = 0; e < 4; ++e) st[e] += __shfl_xor_sync(0xffffffffu, st[e], s);
      if (lane < 4) put_stats(red, c - n0, st, add);
    }
  }
}

// Epilogue of one consumer warpgroup from its 64 x BLOCK_N accumulator in the wgmma fragment
// layout: lane l of warp w holds tile rows 16 w + l / 4 (h = 0) and + 8 (h = 1), columns
// 8 j + 2 (l % 4) + {0, 1} in acc[4 j + 2 h + {0, 1}].  row[h] / row_ok[h]: the global rows.
// red / add: the warp's statistics slots (put_stats), used when p.stats is set.
//
// Tiles inside the output with the common option sets (GELU and two bf16 planes; fp32 with or
// without residual and fused statistics; each with or without bias) take `epilogue_full`.
// Everything else (edge tiles, other plane counts, unaligned tensors) takes the general
// loop below, whose runtime option tests split every column group into short dependent
// branches: measured on H100 at 700 W, it kept one warpgroup 17 us (fp32 store) to 28 us (GELU +
// planes) on a 128 x 128 tile, two to three times the other warpgroup's 8-k-block mainloop.
template <int BLOCK_N>
__device__ __forceinline__ void epilogue(const TcParams& p, const float (&acc)[BLOCK_N / 2],
                                         const long long (&row)[2], const bool (&row_ok)[2], int n0,
                                         int lane, long long out_off, double* red, bool add) {
  const bool vec_r = p.residual != nullptr && (p.ldr & 1) == 0 && (reinterpret_cast<uintptr_t>(p.residual) & 7) == 0;
  const bool vec_o = p.out_f32 != nullptr && (p.ldo & 1) == 0 && (reinterpret_cast<uintptr_t>(p.out_f32) & 7) == 0;
  const bool vec_p = p.out_planes != nullptr && (p.ldp & 1) == 0 && (p.out_plane_stride & 1) == 0 &&
                     (reinterpret_cast<uintptr_t>(p.out_planes) & 3) == 0;
  // the two rows' operands, addressed once (null where the GEMM has no such tensor)
  const float* res_row[2];
  float* out_row[2];
  __nv_bfloat16* pl_row[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    res_row[h] = p.residual != nullptr ? p.residual + row[h] * (long long)p.ldr : nullptr;
    out_row[h] = p.out_f32 != nullptr ? p.out_f32 + out_off + row[h] * (long long)p.ldo : nullptr;
    pl_row[h] = p.out_planes != nullptr ? p.out_planes + row[h] * (long long)p.ldp : nullptr;
  }
  if (p.residual != nullptr) {
    // both rows' residual segments into L1 up front: the loads below then do not each wait on L2
    const int c = n0 + 32 * (lane & 3);
    if ((lane & 3) < BLOCK_N / 32 && c < p.N) {
#pragma unroll
      for (int h = 0; h < 2; ++h)
        if (row_ok[h]) asm volatile("prefetch.global.L1 [%0];" ::"l"(res_row[h] + c));
    }
  }
  if (n0 + BLOCK_N <= p.N && row_ok[0] && row_ok[1]) {
    const bool bias = p.bias != nullptr, resid = p.residual != nullptr, stats = p.stats != nullptr;
#define TAPIR_EPI_FULL(B, G, R, F, PL, S)                                                  \
    if (bias == B && resid == R && stats == S)                                              \
      return epilogue_full<BLOCK_N, B, G, R, F, PL, S>(p, acc, res_row, out_row, pl_row, n0, lane, red, add);
    if (p.act == 1 && !resid && !stats && p.out_f32 == nullptr && p.out_P == 2 && vec_p) {
      TAPIR_EPI_FULL(true, true, false, false, 2, false)
      TAPIR_EPI_FULL(false, true, false, false, 2, false)
    }
    if (p.act == 0 && p.out_planes == nullptr && vec_o && (!resid || vec_r)) {
      TAPIR_EPI_FULL(true, false, true, true, 0, true) TAPIR_EPI_FULL(true, false, true, true, 0, false)
      TAPIR_EPI_FULL(true, false, false, true, 0, true) TAPIR_EPI_FULL(true, false, false, true, 0, false)
      TAPIR_EPI_FULL(false, false, true, true, 0, true) TAPIR_EPI_FULL(false, false, true, true, 0, false)
      TAPIR_EPI_FULL(false, false, false, true, 0, true) TAPIR_EPI_FULL(false, false, false, true, 0, false)
    }
#undef TAPIR_EPI_FULL
  }
#pragma unroll
  for (int j = 0; j < BLOCK_N / 8; ++j) {
    const int c = n0 + 8 * j + 2 * (lane & 3);
    const bool ok0 = c < p.N, ok1 = c + 1 < p.N;
    float b0 = 0.f, b1 = 0.f;
    if (p.bias != nullptr) {
      if (ok0) b0 = __ldg(p.bias + c);
      if (ok1) b1 = __ldg(p.bias + c + 1);
    }
    float st[4] = {0.f, 0.f, 0.f, 0.f};  // column c, c + 1: sum, then sum of squares
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
      if (!row_ok[h] || !ok0) continue;
      if (p.bias != nullptr) { v0 += b0; v1 += b1; }
      if (p.act == 1) { v0 = gelu_tanh(v0); v1 = gelu_tanh(v1); }
      if (p.residual != nullptr) {
        const float* rp = res_row[h] + c;
        if (ok1 && vec_r) {
          const float2 t = *reinterpret_cast<const float2*>(rp);
          v0 += t.x; v1 += t.y;
        } else {
          v0 += rp[0];
          if (ok1) v1 += rp[1];
        }
      }
      if (p.out_f32 != nullptr) {
        float* o = out_row[h] + c;
        if (ok1 && vec_o) {
          *reinterpret_cast<float2*>(o) = make_float2(v0, v1);
        } else {
          o[0] = v0;
          if (ok1) o[1] = v1;
        }
      }
      if (p.stats != nullptr) {
        // InstanceNorm statistics of the tensor this GEMM produces (nets.py:280-286), fused here
        // so the activation is not re-read
        st[0] += v0; st[2] += v0 * v0;
        if (ok1) { st[1] += v1; st[3] += v1 * v1; }
      }
      if (p.out_planes != nullptr) {
        // successive bf16 terms of v: plane q holds bf16(v - sum_{s<q} plane s)
#pragma unroll
        for (int q = 0; q < 3; ++q) {
          if (q == p.out_P) break;
          __nv_bfloat16* o = pl_row[h] + q * p.out_plane_stride + c;
          if (ok1 && vec_p) {
            *reinterpret_cast<uint32_t*>(o) = bf16x2_split(v0, v1);
          } else {
            const __nv_bfloat16 h0 = __float2bfloat16_rn(v0);
            v0 -= __bfloat162float(h0);
            o[0] = h0;
            if (ok1) {
              const __nv_bfloat16 h1 = __float2bfloat16_rn(v1);
              v1 -= __bfloat162float(h1);
              o[1] = h1;
            }
          }
        }
      }
    }
    if (p.stats != nullptr) {
      // sum over the warp's 16 rows: the 8 lanes that share (l % 4) hold the same columns
#pragma unroll
      for (int s = 4; s < 32; s <<= 1)
#pragma unroll
        for (int e = 0; e < 4; ++e) st[e] += __shfl_xor_sync(0xffffffffu, st[e], s);
      // every slot is written (zeros past N or the last row); flush_stats skips columns past N
      if (lane < 4) put_stats(red, c - n0, st, add);
    }
  }
}

// The tile's statistics from the warpgroup's slots `red` (see kStatsSlotBytes): once all four
// warps have put theirs (named barrier `bar`), per column and value the fp64 sum over the warps,
// one atomic each.  The second barrier keeps the warpgroup's next tile from overwriting slots
// that are still being read.
template <int BLOCK_N>
__device__ __forceinline__ void flush_stats(const TcParams& p, const double* red, int n0, int frame, uint32_t bar) {
  ptx::named_bar_sync(bar, 128);
  double* dst = p.stats + ((long long)frame * p.N + n0) * 2;
  for (int i = threadIdx.x & 127; i < 2 * BLOCK_N; i += 128)
    if (n0 + i / 2 < p.N)
      atomicAdd(dst + i, red[i] + red[2 * BLOCK_N + i] + red[4 * BLOCK_N + i] + red[6 * BLOCK_N + i]);
  ptx::named_bar_sync(bar, 128);
}

// Conv m-tile `m_tile` of p.tileW x p.tileH output pixels: its frame and top-left pixel.
struct ConvTile {
  int frame, y0, x0;
};
__device__ __forceinline__ ConvTile conv_tile(const TcParams& p, int m_tile) {
  const int per_frame = p.tiles_x * p.tiles_y;
  const int frame = m_tile / per_frame;
  const int r = m_tile - frame * per_frame;
  return {frame, (r / p.tiles_x) * p.tileH, (r % p.tiles_x) * p.tileW};
}

// Global row of tile row r (0..127) of output tile `m_tile`, and whether it exists; a plain tile's
// problem has m_rows rows.
__device__ __forceinline__ void tile_row(const TcParams& p, int m_tile, int m_rows, int r, long long& row,
                                         bool& ok) {
  if (p.mode == kGemmConv3x3) {
    const ConvTile ct = conv_tile(p, m_tile);
    const int y = ct.y0 + r / p.tileW;
    const int x = ct.x0 + r % p.tileW;
    ok = (y < p.H) && (x < p.W);
    row = ((long long)ct.frame * p.H + y) * p.W + x;
  } else {
    row = (long long)m_tile * kBlockM + r;
    ok = row < m_rows;
  }
}

// Epilogue of rows [r_base, r_base + 64) of output tile `m_tile`, held by one consumer warpgroup;
// `red`: the warpgroup's statistics slots (add: the tile's other half is already in them).
template <int BLOCK_N>
__device__ __forceinline__ void tile_epilogue(const TcParams& p, const float (&acc)[BLOCK_N / 2], int m_tile,
                                              int m_rows, int r_base, int n0, int warp, int lane, long long out_off,
                                              double* red, bool add) {
  const int r0 = r_base + warp * 16 + (lane >> 2);
  long long row[2];
  bool row_ok[2];
  tile_row(p, m_tile, m_rows, r0, row[0], row_ok[0]);
  tile_row(p, m_tile, m_rows, r0 + 8, row[1], row_ok[1]);
  epilogue<BLOCK_N>(p, acc, row, row_ok, n0, lane, out_off, red + warp * 2 * BLOCK_N, add);
}

// The frame of output tile `m_tile` (tiles never straddle frames where statistics are fused).
__device__ __forceinline__ int tile_frame(const TcParams& p, int m_tile) {
  return (p.mode == kGemmConv3x3) ? conv_tile(p, m_tile).frame
                                  : (int)(((long long)m_tile * kBlockM) / p.rows_per_frame);
}

// Whether all rows and columns of output tile (m_tile, n0) exist.  Its 128 rows are consecutive
// output rows wherever the host sets plane_tma: plain mode, or tiles of whole image rows.
template <int BLOCK_N>
__device__ __forceinline__ bool whole_tile(const TcParams& p, int m_tile, int n0) {
  long long last;
  bool ok;
  tile_row(p, m_tile, p.M, kBlockM - 1, last, ok);
  return ok && n0 + BLOCK_N <= p.N;
}

// The GELU + two-plane epilogue of rows [r_base, r_base + 64) of whole tile `m_tile`, with the same
// values as epilogue_full's, written through shared memory.  Register stores write one 4-byte word
// in each of 8 rows per warp instruction, half of every 32-byte sector, and kept the warpgroup in
// its epilogue longer than the other warpgroup's mainloop.  Here, per 64 columns, stmatrix puts
// each plane's 64 x 64 box into its buffer (`boxes`, then + 8 KB; 128B-swizzled as the tensor map
// expects) and one thread writes both boxes out with TMA stores of whole 128-byte rows.  Before
// the warpgroup overwrites the buffers, that thread waits until the previous stores have read
// them.
template <int BLOCK_N, bool BIAS>
__device__ __forceinline__ void epilogue_planes_tma(const TcParams& p, float (&acc)[BLOCK_N / 2], int m_tile,
                                                    int r_base, int n0, uint32_t boxes, uint32_t bar, int warp,
                                                    int lane) {
  const bool issuer = warp == 0 && lane == 0;
  long long row0;
  bool ok;
  tile_row(p, m_tile, p.M, r_base, row0, ok);
  // stmatrix: lanes 8 i .. 8 i + 7 address the rows of matrix i, rows 8 (i & 1) on, column group i >> 1
  const uint32_t rr = lane & 7;
  const uint32_t row_addr = (uint32_t)(16 * warp + 8 * ((lane >> 3) & 1) + rr) * 128;
  const uint32_t chunk_hi = (uint32_t)lane >> 4;
#pragma unroll
  for (int cb = 0; cb < BLOCK_N / 64; ++cb) {
    if (issuer) ptx::bulk_wait_read<0>();
    ptx::named_bar_sync(bar, 128);  // the previous stores have read the buffers
    // the arithmetic below stays after the barrier: with both accumulator halves live, the
    // registers hold one stmatrix worth of plane values at a time
    ptx::reg_fence(acc);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      uint32_t pl[2][4];  // plane q of column group 8 cb + 2 k + g, rows +0 / +8 (s): pl[q][2 g + s]
#pragma unroll
      for (int g = 0; g < 2; ++g) {
        const int j = 8 * cb + 2 * k + g;
        const int c = n0 + 8 * j + 2 * (lane & 3);
        float b0 = 0.f, b1 = 0.f;
        if constexpr (BIAS) { b0 = __ldg(p.bias + c); b1 = __ldg(p.bias + c + 1); }
#pragma unroll
        for (int s = 0; s < 2; ++s) {
          float v0 = acc[4 * j + 2 * s], v1 = acc[4 * j + 2 * s + 1];
          if constexpr (BIAS) { v0 += b0; v1 += b1; }
          v0 = gelu_tanh(v0); v1 = gelu_tanh(v1);
          pl[0][2 * g + s] = bf16x2_split(v0, v1);
          pl[1][2 * g + s] = bf16x2_split(v0, v1);
        }
      }
#pragma unroll
      for (int q = 0; q < 2; ++q)
        ptx::stmatrix_x4(boxes + q * kPlaneBoxBytes + row_addr + (((2 * k + chunk_hi) ^ rr) << 4), pl[q][0],
                         pl[q][1], pl[q][2], pl[q][3]);
    }
    ptx::fence_proxy_async_shared();
    ptx::named_bar_sync(bar, 128);  // both boxes are written
    if (issuer) {
#pragma unroll
      for (int q = 0; q < 2; ++q)
        ptx::tma_store_3d(&p.tmPlanes, boxes + q * kPlaneBoxBytes, n0 + 64 * cb, (int)row0, q);
      ptx::bulk_commit();
    }
  }
}

// The group of linear m-tile `m_tile` of a grouped GEMM: the last g with group_tile0[g] <= m_tile
// (every group has at least one tile).
__device__ __forceinline__ int tile_group(const TcParams& p, int m_tile) {
  int lo = 0, hi = p.groups - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (p.group_tile0[mid] <= m_tile) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

// Work item w in the order (batch or group, m-tile, n-tile, k-slice); m_tile is the tile within its
// batch or group, [kb0, kb1) its k-blocks.  Returns the k-slice.
template <int BLOCK_N>
__device__ __forceinline__ int decode_work(const TcParams& p, int w, int& bat, int& m_tile, int& n0, int& kb0,
                                           int& kb1) {
  const int S = p.split_k;
  const int split = w % S;
  const int tile = w / S;
  m_tile = tile / p.num_n_tiles;
  n0 = (tile - m_tile * p.num_n_tiles) * BLOCK_N;
  if (p.groups > 0) {
    bat = tile_group(p, m_tile);
    m_tile -= p.group_tile0[bat];
  } else {
    bat = m_tile / p.m_tiles_per_batch;
    m_tile -= bat * p.m_tiles_per_batch;
  }
  // 32-bit: num_k_blocks < 2^25 and S <= 8.  A 64-bit division here is a subroutine call, which
  // the ping-pong consumers would pay twice between their epilogue and their next turn.
  kb0 = p.num_k_blocks * split / S;
  kb1 = p.num_k_blocks * (split + 1) / S;
  return split;
}

// Position in a ring of STAGES stages: the stage, and the parity of its current fill.
template <int STAGES>
struct StageCursor {
  int stage = 0;
  uint32_t phase = 0;
  __device__ __forceinline__ void advance() {
    if (++stage == STAGES) { stage = 0; phase ^= 1u; }
  }
  // past n >= 0 positions at once
  __device__ __forceinline__ void advance(int n) {
    stage += n;
    phase ^= (uint32_t)(stage / STAGES) & 1u;
    stage %= STAGES;
  }
};

// A work item as the consumers see it: output tile (m_tile, n0), the offset of its fp32 output
// (k-slice partial buffer and batch or group), its k-blocks [kb0, kb1) and, in plain mode, the rows
// of its problem.
struct Work {
  int m_tile, n0, kb0, kb1;
  long long out_off;
  int m_rows;
};

// The dynamic shared memory from its first 1024-byte boundary: the 128B swizzle of TMA and wgmma
// repeats every 1024 B of absolute address.
__device__ __forceinline__ uint8_t* aligned_smem(uint8_t* smem_raw) {
  return smem_raw + ((1024u - (ptx::smem_u32(smem_raw) & 1023u)) & 1023u);
}

// Thread 0's set-up before the __syncthreads() that follows: the barriers of one or two stage
// rings laid out one after the other at `bars`, each as full[stages] (one arrival: the producer's
// expect_tx) then empty[stages] (`empty_arrivals` each), and a prefetch of the producer's maps.
__device__ __forceinline__ void init_rings(uint64_t* bars, uint32_t empty_arrivals, const CUtensorMap* map_a,
                                           const CUtensorMap* map_b, int stages0, int stages1 = 0) {
  if (threadIdx.x != 0) return;
  const int ring_stages[2] = {stages0, stages1};
  for (const int stages : ring_stages) {
    for (int s = 0; s < stages; ++s) {
      ptx::mbar_init(&bars[s], 1);
      ptx::mbar_init(&bars[stages + s], empty_arrivals);
    }
    bars += 2 * stages;
  }
  ptx::fence_barrier_init();
  ptx::prefetch_tensormap(map_a);
  ptx::prefetch_tensormap(map_b);
}

// The MMAs of one k-block, in the order of every kernel (plane pair (i, j), then k step), into
// HALVES m64 accumulators (A rows 64 h on: eight swizzle atoms, 8 a_sbo bytes, further).  A plane i
// starts at a + i * a_plane with its 8-row swizzle atoms `a_sbo` bytes apart; B plane j at
// b + j * b_plane.
template <int BLOCK_N, int P, int HALVES>
__device__ __forceinline__ void mma_k_block(float (&acc)[HALVES][BLOCK_N / 2], uint32_t a, uint32_t a_plane,
                                            uint32_t a_sbo, uint32_t b, uint32_t b_plane, uint32_t accumulate) {
#pragma unroll
  for (int i = 0; i < P; ++i) {
#pragma unroll
    for (int j = 0; j < P - i; ++j) {
      uint64_t adesc[HALVES];
#pragma unroll
      for (int h = 0; h < HALVES; ++h) adesc[h] = ptx::make_smem_desc_sw128(a + i * a_plane + h * 8 * a_sbo, a_sbo);
      const uint64_t bdesc = ptx::make_smem_desc_sw128(b + j * b_plane);
#pragma unroll
      for (int k = 0; k < kBlockK / kMmaK; ++k) {
#pragma unroll
        for (int h = 0; h < HALVES; ++h) wgmma_bf16<BLOCK_N>(acc[h], adesc[h] + 2 * k, bdesc + 2 * k, accumulate);
        accumulate = 1u;
      }
    }
  }
}

// One consumer k-block: waits for its stage to fill, issues its MMAs as one wgmma group, and
// once the previous k-block's group has retired releases that k-block's stage (empty[prev]; none
// before a tile's first k-block, prev < 0) with one arrival per warp.
template <int BLOCK_N, int P, int HALVES>
__device__ __forceinline__ void consume_k_block(float (&acc)[HALVES][BLOCK_N / 2], uint64_t* full, uint32_t parity,
                                                const TcParams& p, int err_code, uint32_t a, uint32_t a_plane,
                                                uint32_t a_sbo, uint32_t b, uint32_t b_plane, uint32_t accumulate,
                                                uint64_t* empty, int prev, int lane) {
  ptx::mbar_wait(full, parity, p.err, err_code);
  ptx::wgmma_fence();
  mma_k_block<BLOCK_N, P, HALVES>(acc, a, a_plane, a_sbo, b, b_plane, accumulate);
  ptx::wgmma_commit();
  // the previous k-block's MMAs have retired once at most this group is pending
  ptx::wgmma_wait<1>();
#pragma unroll
  for (int h = 0; h < HALVES; ++h) ptx::reg_fence(acc[h]);
  if (prev >= 0 && lane == 0) ptx::mbar_arrive(&empty[prev]);
}

// The operand sources of wgmma_kernel: Ring (both GEMM schedules) and HaloRing (both halo
// convolution schedules).  Each has the same members:
//   kBlockN, kP, kStages     tile width, operand planes, stages of the ring the k-blocks stream through
//   kAPlane, kASbo, kBPlane  A: bytes between planes and between 8-row swizzle atoms; B: between planes
//   kPlaneBoxes              its staging holds epilogue_planes_tma's output boxes
//   kFullErr                 the error code of the consumers' full-barrier wait
//   full_bar, empty_bar      that ring's barriers
//   produce(p)               the TMA producer
//   work(p, w)               work item w: its output tile, output offset and k-blocks
//   kblock(t, stage, kb)     A and B of k-block kb of the CTA's local tile t, held in `stage`
//   wait_tile, release_tile  what a tile needs beside its k-blocks (the halo patch)
//   consumer_staging(cw)     consumer cw's statistics slots or output boxes

// Shared-memory ring of both GEMM schedules: kStages stages of P A planes then P B planes, STAGING
// bytes (1024-aligned) for the epilogue, then the full and empty mbarriers.
template <int BLOCK_N, int P, int STAGING>
struct Ring {
  using Cfg = TcCfg<BLOCK_N, P, STAGING>;
  static_assert(Cfg::kStages == TcCfg<BLOCK_N, P>::kStages, "the epilogue staging must not cost the ring a stage");
  static_assert(kStatsSlotBytes<BLOCK_N> <= STAGING / kConsumers, "each consumer's staging holds its statistics slots");
  static constexpr int kBlockN = BLOCK_N, kP = P, kStages = Cfg::kStages;
  static constexpr uint32_t kAPlane = Cfg::kABytes, kASbo = 1024, kBPlane = Cfg::kBBytes;
  static constexpr bool kPlaneBoxes = STAGING >= kPlaneStagingBytes;
  static constexpr int kFullErr = 103;
  uint8_t* smem;
  uint8_t* staging;
  uint64_t* full_bar;
  uint64_t* empty_bar;
  __device__ __forceinline__ Ring(uint8_t* smem_raw, const TcParams& p, uint32_t empty_arrivals)
      : smem(aligned_smem(smem_raw)),
        staging(smem + Cfg::kStages * Cfg::kStageBytes),
        full_bar(reinterpret_cast<uint64_t*>(staging + STAGING)),
        empty_bar(full_bar + Cfg::kStages) {
    init_rings(full_bar, empty_arrivals, &p.tmA, &p.tmB, Cfg::kStages);
  }

  __device__ __forceinline__ Work work(const TcParams& p, int w) const {
    Work wk;
    int bat;
    const int split = decode_work<BLOCK_N>(p, w, bat, wk.m_tile, wk.n0, wk.kb0, wk.kb1);
    if (p.groups > 0) {
      wk.out_off = split * p.split_stride + (long long)p.group_row0[bat] * p.ldo;
      wk.m_rows = p.group_row0[bat + 1] - p.group_row0[bat];
    } else {
      wk.out_off = split * p.split_stride + bat * p.out_batch_stride;
      wk.m_rows = p.M;
    }
    return wk;
  }
  __device__ __forceinline__ void kblock(int, int stage, int, uint32_t& a, uint32_t& b) const {
    a = ptx::smem_u32(smem + stage * Cfg::kStageBytes);
    b = a + P * Cfg::kABytes;
  }
  __device__ __forceinline__ void wait_tile(const TcParams&, int) const {}
  __device__ __forceinline__ void release_tile(int) const {}
  __device__ __forceinline__ uint8_t* consumer_staging(int cw) const { return staging + cw * (STAGING / kConsumers); }

  // TMA producer (one thread): the k-blocks of this CTA's work items, in order, into the ring.
  __device__ __forceinline__ void produce(const TcParams& p) const {
    const int num_work = p.num_m_tiles * p.num_n_tiles * p.split_k;
    StageCursor<Cfg::kStages> cur;
    for (int w = blockIdx.x; w < num_work; w += gridDim.x) {
      int bat, m_tile, n0, kb0, kb1;
      decode_work<BLOCK_N>(p, w, bat, m_tile, n0, kb0, kb1);
      // batch or group = row offset into the flattened operands; rows loaded past the end of a
      // batch or group belong to the next one (or are TMA zero fill) and are masked by the epilogue
      const int a_row0 = (p.groups > 0 ? p.group_row0[bat] : (int)(bat * p.a_batch_rows)) + m_tile * kBlockM;
      const int b_row0 = (int)(bat * p.b_batch_rows) + n0;
      ConvTile ct{0, 0, 0};
      if (p.mode == kGemmConv3x3) ct = conv_tile(p, m_tile);
      for (int kb = kb0; kb < kb1; ++kb) {
        ptx::mbar_wait(&empty_bar[cur.stage], cur.phase ^ 1u, p.err, 101);
        ptx::mbar_arrive_expect_tx(&full_bar[cur.stage], Cfg::kStageBytes);
        uint8_t* sa = smem + cur.stage * Cfg::kStageBytes;
        uint8_t* sb = sa + P * Cfg::kABytes;
        if (p.mode == kGemmConv3x3) {
          const int tap = kb / p.cblocks;
          const int cb = kb - tap * p.cblocks;
          const int ky = tap / 3, kx = tap - ky * 3;
#pragma unroll
          for (int pl = 0; pl < P; ++pl)
            ptx::tma_load_5d(sa + pl * Cfg::kABytes, &p.tmA, &full_bar[cur.stage], cb * kBlockK,
                             ct.x0 + kx - 1, ct.y0 + ky - 1, ct.frame, pl);
        } else {
#pragma unroll
          for (int pl = 0; pl < P; ++pl)
            ptx::tma_load_3d(sa + pl * Cfg::kABytes, &p.tmA, &full_bar[cur.stage], kb * kBlockK,
                             a_row0, pl);
        }
#pragma unroll
        for (int pl = 0; pl < P; ++pl)
          ptx::tma_load_3d(sb + pl * Cfg::kBBytes, &p.tmB, &full_bar[cur.stage], kb * kBlockK, b_row0, pl);
        cur.advance();
      }
    }
  }
};

// ------------------------------------------------------------------------------ halo-patch conv
// 3x3 convolution, C = 64 -> N = 64 (the first ResNet group, stride 1).  The generic implicit GEMM
// loads one shifted 128-pixel box per tap, so every input element crosses L2 -> SM nine times.
// Here a tile of 8 x 16 output pixels stages its 10 x 18 input patch ONCE (18 TMA loads of one
// patch row each into rows padded to 16 pixels = 2048 B, so that every 8-pixel group of every tap
// view has the same swizzle phase) and the nine taps are nine shared-memory views of it: output
// rows 8c .. 8c + 7 of the tile (one m64 wgmma) read start = patch + (8c + ky) * 2048 + kx * 128,
// with 2048 B between their 8-pixel row groups.  B (weights, 8 KB per tap and plane) streams
// through a 4-slot ring, one tap per k-block.  Both schedules of wgmma_kernel run it:
// conv3x3_halo_kernel and conv3x3_halo_pingpong_kernel.
constexpr int kHaloTileW = 8, kHaloTileH = 16;
constexpr int kHaloRowBytes = 2048;                        // 16 pixels x 128 B
constexpr int kHaloPatchRows = kHaloTileH + 2;
constexpr int kHaloPatchBytes = kHaloPatchRows * kHaloRowBytes;  // per plane
constexpr int kHaloRowLoadBytes = (kHaloTileW + 2) * 128;  // what one TMA row load delivers
constexpr int kHaloPatchStages = 2;
constexpr int kHaloBStages = 4;
constexpr int kHaloBBytes = 64 * 128;                      // per plane and tap
constexpr int kHaloStatsBytes = kConsumers * kStatsSlotBytes<64>;
template <int P>
struct HaloCfg {
  static constexpr int kPatchStage = P * kHaloPatchBytes;
  static constexpr int kBStage = P * kHaloBBytes;
  static constexpr int kSmemBytes =
      1024 + kHaloPatchStages * kPatchStage + kHaloBStages * kBStage + kHaloStatsBytes + kBarrierBytes;
  static_assert(kSmemBytes <= kSmemLimit, "halo conv: the rings and the statistics slots must fit as they are");
};

// Shared memory of both halo schedules: the patch ring [2][P][18][2048], the B ring [4][P][64][128],
// the consumers' statistics slots, then the full / empty barriers of the two rings.  The k-blocks
// (full_bar, empty_bar) are the B ring's.
template <int P>
struct HaloRing {
  using Cfg = HaloCfg<P>;
  static constexpr int kBlockN = 64, kP = P, kStages = kHaloBStages;
  static constexpr uint32_t kAPlane = kHaloPatchBytes, kASbo = kHaloRowBytes, kBPlane = kHaloBBytes;
  static constexpr bool kPlaneBoxes = false;
  static constexpr int kFullErr = 405;
  uint8_t* patch;
  uint8_t* bring;
  uint8_t* staging;
  uint64_t* pfull;      // [2]
  uint64_t* pempty;     // [2]
  uint64_t* full_bar;   // [4]
  uint64_t* empty_bar;  // [4]
  __device__ __forceinline__ HaloRing(uint8_t* smem_raw, const TcParams& p, uint32_t empty_arrivals) {
    patch = aligned_smem(smem_raw);
    bring = patch + kHaloPatchStages * Cfg::kPatchStage;
    staging = bring + kHaloBStages * Cfg::kBStage;
    pfull = reinterpret_cast<uint64_t*>(staging + kHaloStatsBytes);
    pempty = pfull + kHaloPatchStages;
    full_bar = pempty + kHaloPatchStages;
    empty_bar = full_bar + kHaloBStages;
    init_rings(pfull, empty_arrivals, &p.tmPatch, &p.tmB, kHaloPatchStages, kHaloBStages);
  }

  // TMA producer (one thread): per tile of this CTA, its patch, then its nine taps of B.
  __device__ __forceinline__ void produce(const TcParams& p) const {
    StageCursor<kHaloPatchStages> pc;
    StageCursor<kHaloBStages> bc;
    for (int w = blockIdx.x; w < p.num_m_tiles; w += gridDim.x) {
      const ConvTile ct = conv_tile(p, w);
      ptx::mbar_wait(&pempty[pc.stage], pc.phase ^ 1u, p.err, 401);
      ptx::mbar_arrive_expect_tx(&pfull[pc.stage], (uint32_t)(P * kHaloPatchRows * kHaloRowLoadBytes));
      for (int pl = 0; pl < P; ++pl)
        for (int pr = 0; pr < kHaloPatchRows; ++pr)
          ptx::tma_load_5d(patch + pc.stage * Cfg::kPatchStage + pl * kHaloPatchBytes + pr * kHaloRowBytes,
                           &p.tmPatch, &pfull[pc.stage], 0, ct.x0 - 1, ct.y0 - 1 + pr, ct.frame, pl);
      pc.advance();
      for (int tap = 0; tap < 9; ++tap) {
        ptx::mbar_wait(&empty_bar[bc.stage], bc.phase ^ 1u, p.err, 402);
        ptx::mbar_arrive_expect_tx(&full_bar[bc.stage], (uint32_t)Cfg::kBStage);
#pragma unroll
        for (int pl = 0; pl < P; ++pl)
          ptx::tma_load_3d(bring + bc.stage * Cfg::kBStage + pl * kHaloBBytes, &p.tmB, &full_bar[bc.stage],
                           tap * kBlockK, 0, pl);
        bc.advance();
      }
    }
  }

  __device__ __forceinline__ Work work(const TcParams&, int w) const { return {w, 0, 0, 9, 0, 0}; }
  // tap kb = 3 ky + kx: the patch view of output rows 0-7 (see above)
  __device__ __forceinline__ void kblock(int t, int stage, int kb, uint32_t& a, uint32_t& b) const {
    const int ky = kb / 3, kx = kb - ky * 3;
    a = ptx::smem_u32(patch + (t % kHaloPatchStages) * Cfg::kPatchStage) + ky * kHaloRowBytes + kx * 128;
    b = ptx::smem_u32(bring + stage * Cfg::kBStage);
  }
  // The producer fills the patch stages in tile order: local tile t's patch is fill t / 2 of stage t % 2.
  __device__ __forceinline__ void wait_tile(const TcParams& p, int t) const {
    ptx::mbar_wait(&pfull[t % kHaloPatchStages], (uint32_t)(t / kHaloPatchStages) & 1u, p.err, 404);
  }
  __device__ __forceinline__ void release_tile(int t) const { ptx::mbar_arrive(&pempty[t % kHaloPatchStages]); }
  __device__ __forceinline__ uint8_t* consumer_staging(int cw) const { return staging + cw * kStatsSlotBytes<64>; }
};

// ------------------------------------------------------------------------------ the kernels
// Named barriers 1, 2: consumer 0's, consumer 1's turn (ping-pong).  3, 4: their epilogue staging
// (output boxes or statistics).
constexpr uint32_t kTurnBarrier = 1;
constexpr uint32_t kStagingBarrier = 3;
// setmaxnreg: registers of the producer and of each consumer warpgroup thread.  The consumers of
// the ping-pong kernels hold 128 accumulators per thread at BLOCK_N = 128; the cooperative
// kernel's straight-line epilogue with statistics spilled at the 168 registers of an even split.
constexpr int kProducerRegs = 40;
constexpr int kConsumerRegs = 232;

// The body of every wgmma kernel, over the operand source Src (Ring or HaloRing) in one of two
// schedules.  Warpgroup 0's first thread runs Src's producer; warpgroups 1 and 2 consume:
//   cooperative (PINGPONG false): both consumers work on every tile, consumer cw on its rows
//     64 cw .. 64 cw + 63 (one m64 accumulator, A from + 8 cw kASbo), and they run their epilogues
//     at the same time.  Used for split-K, P = 3 and where a CTA gets too few tiles for
//     ping-pong (pick_pingpong, launch_halo).
//   ping-pong: consumer cw owns the CTA's local tiles t with t % 2 == cw, whole (two m64
//     accumulators, rows 0-63 and 64-127).  The warpgroups take turns on the tensor pipe: one
//     issues its tile's whole mainloop, passes the turn and runs its epilogue while the other's
//     MMAs execute, so the epilogue costs no MMA time as long as it is shorter than a mainloop.
//
// Each consumer walks every local tile of its CTA in order, as the producer fills the ring, and
// keeps one ring position, advanced by each tile's k-block count; under ping-pong it only
// advances it over the other warpgroup's tiles.  A full-barrier parity wait is exact when every
// earlier fill of the stage has completed (the producer cannot be a fill ahead: it waits for the
// stage to be released).  The cooperative consumers wait on every position in order.  Under
// ping-pong, a warpgroup waits on its tile's first stage only after the other has passed the
// turn, that is after it has waited on every stage of the tile before; by induction every earlier
// position has been waited on.  The halo patch ring holds one tile per stage and follows the same
// argument: under ping-pong consumer cw always reads patch stage cw.
//
// Every output element sums its K terms in the same order in both schedules, so they give
// bit-identical outputs (the fused statistics keep the per-warp fp32 partials as well; only the
// order of their fp64 additions differs, as the order of the atomics may between two runs of
// either kernel).
template <class Src, bool PINGPONG>
__device__ __forceinline__ void wgmma_kernel(const TcParams& p) {
  constexpr int BLOCK_N = Src::kBlockN, HALVES = PINGPONG ? 2 : 1;
  constexpr bool kBoxes = PINGPONG && Src::kPlaneBoxes;
  extern __shared__ uint8_t smem_raw[];
  const Src src(smem_raw, p, PINGPONG ? 4 : kConsumerArrivals);  // one arrive per reading warp

  const int wg = threadIdx.x >> 7;
  const int warp = (threadIdx.x >> 5) & 3;  // within the warpgroup
  const int lane = threadIdx.x & 31;
  __syncthreads();

  if (wg == 0) {
    ptx::setmaxnreg_dec<kProducerRegs>();
    if (threadIdx.x == 0) src.produce(p);
    return;
  }
  ptx::setmaxnreg_inc<kConsumerRegs>();

  const int cw = wg - 1;
  const uint32_t a_rows = PINGPONG ? 0u : (uint32_t)cw * 8 * Src::kASbo;
  uint8_t* const staging = src.consumer_staging(cw);
  double* const red = reinterpret_cast<double*>(staging);
  // split-K (small problems that cannot fill the GPU): work item = (tile, k-slice)
  const int num_work = p.num_m_tiles * p.num_n_tiles * p.split_k;
  const int my_tiles = (num_work - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;
  StageCursor<Src::kStages> cur;
  float acc[HALVES][BLOCK_N / 2];
  for (int t = 0; t < my_tiles; ++t) {
    const Work wk = src.work(p, (int)blockIdx.x + t * (int)gridDim.x);
    if (PINGPONG && (t & 1) != cw) {
      cur.advance(wk.kb1 - wk.kb0);
      continue;
    }
    if (PINGPONG && t > 0) ptx::named_bar_sync(kTurnBarrier + cw, 256);
#pragma unroll
    for (int h = 0; h < HALVES; ++h)
#pragma unroll
      for (int i = 0; i < BLOCK_N / 2; ++i) acc[h][i] = 0.f;
    src.wait_tile(p, t);
    int prev = -1;
    for (int kb = wk.kb0; kb < wk.kb1; ++kb) {
      uint32_t a, b;
      src.kblock(t, cur.stage, kb, a, b);
      consume_k_block<BLOCK_N, Src::kP, HALVES>(acc, &src.full_bar[cur.stage], cur.phase, p, Src::kFullErr,
                                                a + a_rows, Src::kAPlane, Src::kASbo, b, Src::kBPlane, kb > wk.kb0,
                                                src.empty_bar, prev, lane);
      prev = cur.stage;
      cur.advance();
    }
    // every MMA of this tile is issued: the other warpgroup's tile, if it has one, may start
    if (PINGPONG && t + 1 < my_tiles) ptx::named_bar_arrive(kTurnBarrier + (1 - cw), 256);
    ptx::wgmma_wait<0>();
#pragma unroll
    for (int h = 0; h < HALVES; ++h) ptx::reg_fence(acc[h]);
    if (lane == 0) {
      if (prev >= 0) ptx::mbar_arrive(&src.empty_bar[prev]);
      src.release_tile(t);
    }
    const bool staged = kBoxes && p.plane_tma && whole_tile<BLOCK_N>(p, wk.m_tile, wk.n0);
    // one copy of the epilogue code for both ping-pong halves: it runs while the other
    // warpgroup's mainloop executes from the same instruction cache
#pragma unroll 1
    for (int h = 0; h < HALVES; ++h) {
      const int r_base = 64 * (PINGPONG ? h : cw);
      if (staged) {
        if constexpr (kBoxes) {  // only the ping-pong GEMM compiles this path
          const uint32_t boxes = ptx::smem_u32(staging);
          if (p.bias != nullptr)
            epilogue_planes_tma<BLOCK_N, true>(p, acc[0], wk.m_tile, r_base, wk.n0, boxes, kStagingBarrier + cw,
                                               warp, lane);
          else
            epilogue_planes_tma<BLOCK_N, false>(p, acc[0], wk.m_tile, r_base, wk.n0, boxes, kStagingBarrier + cw,
                                                warp, lane);
        }
      } else {
        tile_epilogue<BLOCK_N>(p, acc[0], wk.m_tile, wk.m_rows, r_base, wk.n0, warp, lane, wk.out_off, red,
                               h == 1);
      }
      if constexpr (HALVES == 2) {
        if (h == 0) {
#pragma unroll
          for (int i = 0; i < BLOCK_N / 2; ++i) acc[0][i] = acc[1][i];
        }
      }
    }
    if (p.stats != nullptr) flush_stats<BLOCK_N>(p, red, wk.n0, tile_frame(p, wk.m_tile), kStagingBarrier + cw);
    // after the warpgroup's last tile: its stores complete while the shared memory still exists
    // (here rather than after the loop, where the BN = 128 instances spill)
    if constexpr (kBoxes)
      if (t + 2 >= my_tiles && warp == 0 && lane == 0) ptx::bulk_wait<0>();
  }
}

// Cooperative GEMM: each warpgroup's statistics slots follow the ring.
template <int BLOCK_N>
constexpr int kCoopStaging = kConsumers * kStatsSlotBytes<BLOCK_N>;

template <int BLOCK_N, int P>
__global__ void __launch_bounds__(kThreads, 1)
gemm_tc_kernel(const __grid_constant__ TcParams p) {
  wgmma_kernel<Ring<BLOCK_N, P, kCoopStaging<BLOCK_N>>, false>(p);
}

// Ping-pong GEMM (no split-K, P <= 2): each warpgroup's two output box buffers follow the ring; a
// tile's statistics slots share them (a GEMM with statistics has no plane output).
template <int BLOCK_N, int P>
__global__ void __launch_bounds__(kThreads, 1)
gemm_tc_pingpong_kernel(const __grid_constant__ TcParams p) {
  static_assert(P <= 2, "ping-pong: P = 3 stays cooperative");
  wgmma_kernel<Ring<BLOCK_N, P, kPlaneStagingBytes>, true>(p);
}

template <int P>
__global__ void __launch_bounds__(kThreads, 1)
conv3x3_halo_kernel(const __grid_constant__ TcParams p) {
  wgmma_kernel<HaloRing<P>, false>(p);
}

template <int P>
__global__ void __launch_bounds__(kThreads, 1)
conv3x3_halo_pingpong_kernel(const __grid_constant__ TcParams p) {
  wgmma_kernel<HaloRing<P>, true>(p);
}

// Second pass of a split-K GEMM: sums the k-slice partials in a fixed order (deterministic) and
// applies the epilogue (bias, GELU, residual, fp32 / bf16-plane outputs).
__global__ void __launch_bounds__(256) splitk_reduce_kernel(const float* __restrict__ part, int S,
                                                            long long split_stride, int ldw,
                                                            const TcParams p) {
  const int groups = (p.N + 3) / 4;
  const long long total = (long long)p.M * groups;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long row = i / groups;
    const int col = (int)(i - row * groups) * 4;
    float x[4] = {0.f, 0.f, 0.f, 0.f};
    for (int s = 0; s < S; ++s) {
      const float4 t = *reinterpret_cast<const float4*>(part + s * split_stride + row * ldw + col);
      x[0] += t.x; x[1] += t.y; x[2] += t.z; x[3] += t.w;
    }
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      if (col + e >= p.N) continue;
      float v = x[e];
      if (p.bias != nullptr) v += p.bias[col + e];
      if (p.act == 1) v = gelu_tanh(v);
      if (p.residual != nullptr) v += p.residual[row * p.ldr + col + e];
      if (p.out_f32 != nullptr) p.out_f32[row * p.ldo + col + e] = v;
      if (p.out_planes != nullptr) {
        for (int q = 0; q < p.out_P; ++q) {
          const __nv_bfloat16 h = __float2bfloat16_rn(v);
          v -= __bfloat162float(h);
          p.out_planes[q * p.out_plane_stride + row * p.ldp + col + e] = h;
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------ host side

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres);
    if (e == cudaSuccess && qres == cudaDriverEntryPointSuccess) fn = reinterpret_cast<EncodeTiledFn>(ptr);
  }
  return fn;
}

int encode_bf16_map(CUtensorMap* m, const void* base, int rank, const cuuint64_t* dims,
                    const cuuint64_t* strides_bytes, const cuuint32_t* box, const char* what) {
  EncodeTiledFn fn = get_encode_fn();
  if (fn == nullptr) {
    set_error("cuTensorMapEncodeTiled entry point not available (driver too old?)");
    return kCudaError;
  }
  cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, (cuuint32_t)rank, const_cast<void*>(base),
                  dims, strides_bytes, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled(%s) failed with CUresult %d (base=%p rank=%d dims=%llu,%llu,%llu "
              "stride0=%llu box=%u,%u,%u)",
              what, (int)r, base, rank, (unsigned long long)dims[0], (unsigned long long)dims[1],
              (unsigned long long)dims[2], (unsigned long long)strides_bytes[0], box[0], box[1], box[2]);
    return kCudaError;
  }
  return kOk;
}

int* device_error_flag() {
  static int* flag[kMaxDevices] = {};
  const int dev = current_device();
  if (flag[dev] == nullptr) {
    if (cudaMalloc(&flag[dev], sizeof(int)) != cudaSuccess) return nullptr;
    cudaMemset(flag[dev], 0, sizeof(int));
  }
  return flag[dev];
}

void choose_conv_tile(int H, int W, int* tw, int* th) {
  long long best = -1;
  for (int w = 128; w >= 8; w >>= 1) {
    const int h = 128 / w;
    const long long tiles = (long long)ceil_div(W, w) * ceil_div(H, h);
    if (best < 0 || tiles < best) { best = tiles; *tw = w; *th = h; }
  }
}

// Map of a row-major operand: P planes of `rows` rows of K elements, `ld` apart, planes
// `plane_stride` apart (0: rows * ld), read in boxes of 64 k x `box_rows` rows of one plane.
int encode_rows_map(CUtensorMap* m, const __nv_bfloat16* base, int K, long long rows, int ld,
                    long long plane_stride, int P, int box_rows, const char* what) {
  const long long plane = plane_stride > 0 ? plane_stride : rows * ld;
  const cuuint64_t dims[3] = {(cuuint64_t)K, (cuuint64_t)rows, (cuuint64_t)P};
  const cuuint64_t str[2] = {(cuuint64_t)ld * 2, (cuuint64_t)plane * 2};
  const cuuint32_t box[3] = {(cuuint32_t)kBlockK, (cuuint32_t)box_rows, 1};
  return encode_bf16_map(m, base, 3, dims, str, box, what);
}

// Map of a conv GEMM's A, the NHWC activation: P planes of [frames][H][W][C] (planes
// a_plane_stride apart, 0: M * C), read in boxes of 64 channels x box_w x box_h pixels of one
// frame and plane.
int encode_nhwc_map(CUtensorMap* m, const GemmArgs& g, int box_w, int box_h, const char* what) {
  const long long plane = g.a_plane_stride > 0 ? g.a_plane_stride : (long long)g.M * g.C;
  const cuuint64_t dims[5] = {(cuuint64_t)g.C, (cuuint64_t)g.W, (cuuint64_t)g.H, (cuuint64_t)g.frames,
                              (cuuint64_t)g.planes};
  const cuuint64_t str[4] = {(cuuint64_t)g.C * 2, (cuuint64_t)g.W * g.C * 2, (cuuint64_t)g.H * g.W * g.C * 2,
                             (cuuint64_t)plane * 2};
  const cuuint32_t box[5] = {(cuuint32_t)kBlockK, (cuuint32_t)box_w, (cuuint32_t)box_h, 1, 1};
  return encode_bf16_map(m, g.a, 5, dims, str, box, what);
}

// Launches a wgmma kernel on at most one CTA per SM over p's work items, timed under the GEMM's
// profiling tag with its FLOPs and algorithmic bytes.  The kernel's shared-memory limit is
// raised once per device.
template <void (*KERNEL)(TcParams), int SMEM_BYTES>
int launch(const char* name, const TcParams& p, const GemmArgs& g, cudaStream_t stream) {
  static PerDeviceOnce configured;
  if (configured.pending()) {
    TAPIR_CUDA(cudaFuncSetAttribute(KERNEL, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
    configured.mark();
  }
  const double kl = g.k_logical > 0 ? g.k_logical : g.K;
  const double out_b = (g.out_f32 ? 4.0 : 0.0) + (g.out_planes ? 2.0 * g.out_P : 0.0) + (g.residual ? 4.0 : 0.0);
  const double a_elems = (g.mode == kGemmConv3x3) ? (double)g.M * g.C : (double)g.M * g.K;
  ProfileScope ps(g.tag ? g.tag : "gemm", stream, 2.0 * g.batch * g.M * g.N * kl,
                  g.batch * (2.0 * g.planes * (a_elems + (double)g.N * g.K) + out_b * g.M * g.N));
  const int sms = num_sms();
  const int work = p.num_m_tiles * p.num_n_tiles * p.split_k;
  KERNEL<<<work < sms ? work : sms, kThreads, SMEM_BYTES, stream>>>(p);
  count_launch();
  TAPIR_LAUNCH_CHECK(name);
  return kOk;
}

template <int BLOCK_N, int P>
int launch_gemm(bool pingpong, const TcParams& p, const GemmArgs& g, cudaStream_t stream) {
  if constexpr (P <= 2)
    if (pingpong)
      return launch<gemm_tc_pingpong_kernel<BLOCK_N, P>, TcCfg<BLOCK_N, P, kPlaneStagingBytes>::kSmemBytes>(
          "gemm_tc_pingpong_kernel", p, g, stream);
  return launch<gemm_tc_kernel<BLOCK_N, P>, TcCfg<BLOCK_N, P, kCoopStaging<BLOCK_N>>::kSmemBytes>("gemm_tc_kernel", p,
                                                                                                 g, stream);
}

// The GEMM kernel for tile width `bn` and g.planes; ping-pong only where pick_pingpong chose it.
int launch_gemm(int bn, bool pingpong, const TcParams& p, const GemmArgs& g, cudaStream_t stream) {
  const int P = g.planes;
  if (bn == 64 && P == 1) return launch_gemm<64, 1>(pingpong, p, g, stream);
  if (bn == 64 && P == 2) return launch_gemm<64, 2>(pingpong, p, g, stream);
  if (bn == 64 && P == 3) return launch_gemm<64, 3>(pingpong, p, g, stream);
  if (bn == 128 && P == 1) return launch_gemm<128, 1>(pingpong, p, g, stream);
  if (bn == 128 && P == 2) return launch_gemm<128, 2>(pingpong, p, g, stream);
  if (bn == 128 && P == 3) return launch_gemm<128, 3>(pingpong, p, g, stream);
  set_error("gemm_tc: no kernel for BLOCK_N=%d planes=%d", bn, P);
  return kUnsupported;
}

// Ping-pong hides a tile's epilogue behind the other warpgroup's mainloop.  It needs at least two
// tiles per CTA, and measured on H100 it loses to the cooperative kernel when CTAs get fewer than
// four tiles of short (< 16 k-block) mainloops: mixer linear_in / linear_out, 2.9 tiles of 8-9
// k-blocks, ran 10-22 % slower.  Split-K work items, P = 3 and batched GEMMs (only the P = 3 cost
// volume is batched or grouped) stay cooperative.  Elsewhere, and in the halo convolution (launch_halo),
// TAPIR_B200_GEMM_SCHEDULE (sw.schedule) forces either schedule.
bool pick_pingpong(int tiles, int num_k_blocks, int P, bool batched, const GemmSwitches& sw) {
  if (P > 2 || batched) return false;
  if (sw.schedule != 0) return sw.schedule == 2;
  const int sms = num_sms();
  return tiles >= 2 * sms && (tiles >= 4 * sms || num_k_blocks >= 16);
}

// Whole ping-pong tiles with tanh-GELU and two bf16 output planes and nothing else (mixer `up`, the
// ExtraConv expansion) write their planes with TMA stores (epilogue_planes_tma) where a tile's rows
// are consecutive output rows and the planes meet TMA's 16-byte rules.  The cooperative schedule
// writes the same tiles with register stores (epilogue_full), the same bits.
int plane_store_params(const GemmArgs& g, bool pingpong, TcParams* p) {
  if (!pingpong) return kOk;
  if (g.act != 1 || g.out_planes == nullptr || g.out_P != 2 || g.out_f32 != nullptr || g.residual != nullptr ||
      g.stats != nullptr)
    return kOk;
  if (g.mode == kGemmConv3x3 && p->tileW != g.W) return kOk;
  if (g.ldp % 8 != 0 || g.out_plane_stride <= 0 || g.out_plane_stride % 8 != 0 ||
      (reinterpret_cast<uintptr_t>(g.out_planes) & 15) != 0)
    return kOk;
  TAPIR_RETURN_IF(encode_rows_map(&p->tmPlanes, g.out_planes, g.N, g.M, g.ldp, g.out_plane_stride, 2, 64, "planes"));
  p->plane_tma = 1;
  return kOk;
}

// Small problems (streaming: one frame, ~1000 mixer rows) cannot fill the GPU with 128 x 128
// tiles: mixer `down` at 1024 rows is 32 tiles for 132 SMs, each walking all of K.
bool small_problem(int m_tiles, int N) {
  return m_tiles * ceil_div(N, 128) * 10 < num_sms() * 6;  // fewer than ~0.6 CTAs per SM
}

// 64-wide tiles for N <= 64, and for small problems when that gives every SM a tile: twice the
// CTAs, each with half the MMA work per k-block.  (The K-summation order of an output element does
// not depend on the tile shape, so results stay bit-identical across these choices.)  A small
// problem that will be split over K keeps 128-wide tiles: the parallelism comes from K, and wide
// tiles re-read the A operand half as often.  TAPIR_B200_BLOCK_N (sw.block_n) forces the width.
int pick_block_n(int m_tiles, int N, bool split_k, const GemmSwitches& sw) {
  if (sw.block_n != 0) return sw.block_n;
  if (N <= 64) return 64;
  if (small_problem(m_tiles, N) && m_tiles * ceil_div(N, 128) * 2 <= num_sms()) return split_k ? 128 : 64;
  return 128;
}

// The parameters every kernel shares: problem, epilogue, batch layout, the generic conv tiling
// and the A map.
int common_params(const GemmArgs& g, TcParams* p) {
  memset(p, 0, sizeof(*p));
  p->M = g.M;
  p->N = g.N;
  p->num_k_blocks = g.K / kBlockK;
  p->frames = g.frames;
  p->mode = g.mode;
  p->bias = g.bias;
  p->residual = g.residual;
  p->ldr = g.ldr;
  p->act = g.act;
  p->out_f32 = g.out_f32;
  p->ldo = g.ldo;
  p->out_planes = g.out_planes;
  p->ldp = g.ldp;
  p->out_plane_stride = g.out_plane_stride;
  p->out_P = g.out_P;
  p->err = device_error_flag();
  p->stats = g.stats;
  p->rows_per_frame = g.rows_per_frame > 0 ? g.rows_per_frame : g.M;
  p->a_batch_rows = g.a_batch_rows > 0 ? g.a_batch_rows : g.M;
  p->b_batch_rows = g.b_batch_rows > 0 ? g.b_batch_rows : g.N;
  p->out_batch_stride = g.out_batch_stride > 0 ? g.out_batch_stride : (long long)g.M * g.ldo;
  p->split_k = 1;
  if (g.mode == kGemmConv3x3) {
    choose_conv_tile(g.H, g.W, &p->tileW, &p->tileH);
    p->H = g.H;
    p->W = g.W;
    p->cblocks = g.C / kBlockK;
    p->tiles_x = ceil_div(g.W, p->tileW);
    p->tiles_y = ceil_div(g.H, p->tileH);
    p->num_m_tiles = g.frames * p->tiles_x * p->tiles_y;
    TAPIR_RETURN_IF(encode_nhwc_map(&p->tmA, g, p->tileW, p->tileH, "A/conv"));
  } else if (g.groups > 0) {
    p->groups = g.groups;
    for (int i = 0; i < g.groups; ++i) {
      p->group_row0[i] = g.group_row0[i];
      p->group_tile0[i + 1] = p->group_tile0[i] + ceil_div(g.group_row0[i + 1] - g.group_row0[i], kBlockM);
    }
    p->group_row0[g.groups] = g.group_row0[g.groups];
    p->num_m_tiles = p->group_tile0[g.groups];
    TAPIR_RETURN_IF(encode_rows_map(&p->tmA, g.a, g.K, g.M, g.lda, g.a_plane_stride, g.planes, kBlockM, "A"));
  } else {
    p->num_m_tiles = ceil_div(g.M, kBlockM) * g.batch;
    TAPIR_RETURN_IF(encode_rows_map(&p->tmA, g.a, g.K, (g.batch - 1) * p->a_batch_rows + g.M, g.lda,
                                    g.a_plane_stride, g.planes, kBlockM, "A"));
  }
  p->m_tiles_per_batch = p->num_m_tiles / g.batch;
  return kOk;
}

// Halo-patch kernel for the C = 64 -> 64 3x3 layers (first ResNet group), see conv3x3_halo_kernel.
// TAPIR_B200_CONV_HALO=0 (sw.halo false): generic path.
bool use_halo(const GemmArgs& g, const GemmSwitches& sw) {
  return sw.halo && g.mode == kGemmConv3x3 && g.C == 64 && g.N == 64 && g.planes <= 2 && g.out_planes == nullptr;
}

// Ping-pong wherever a CTA gets at least two tiles (the clip's 48 frames at 128 x 128: 6144 tiles);
// the single-frame streaming passes (128 tiles) stay cooperative.  TAPIR_B200_GEMM_SCHEDULE
// (sw.schedule) forces either schedule.
int launch_halo(TcParams p, const GemmArgs& g, const GemmSwitches& sw, cudaStream_t stream) {
  p.tileW = kHaloTileW;
  p.tileH = kHaloTileH;
  p.tiles_x = ceil_div(g.W, kHaloTileW);
  p.tiles_y = ceil_div(g.H, kHaloTileH);
  p.num_m_tiles = g.frames * p.tiles_x * p.tiles_y;
  p.num_n_tiles = 1;
  const bool pingpong = sw.schedule != 0 ? sw.schedule == 2 : p.num_m_tiles >= 2 * num_sms();
  TAPIR_RETURN_IF(encode_nhwc_map(&p.tmPatch, g, kHaloTileW + 2, 1, "A/patch"));
  TAPIR_RETURN_IF(encode_rows_map(&p.tmB, g.b, g.K, g.N, g.ldb, g.b_plane_stride, g.planes, 64, "B/halo"));
  if (pingpong) {
    if (g.planes == 1)
      return launch<conv3x3_halo_pingpong_kernel<1>, HaloCfg<1>::kSmemBytes>("conv3x3_halo_pingpong_kernel", p, g, stream);
    return launch<conv3x3_halo_pingpong_kernel<2>, HaloCfg<2>::kSmemBytes>("conv3x3_halo_pingpong_kernel", p, g, stream);
  }
  if (g.planes == 1) return launch<conv3x3_halo_kernel<1>, HaloCfg<1>::kSmemBytes>("conv3x3_halo_kernel", p, g, stream);
  return launch<conv3x3_halo_kernel<2>, HaloCfg<2>::kSmemBytes>("conv3x3_halo_kernel", p, g, stream);
}

// Split-K (deterministic two-pass, below) for problems that cannot half-fill the GPU.  Only where
// the caller allows it by passing a workspace (single-frame streaming steps) and K >= 2048 (mixer
// `down` at ~1000 rows, the ExtraConvs of one frame).  The summation order of a split GEMM
// depends on the row count; offline clips keep the exact chunk / permutation / shard invariance
// (tests/test_properties_gpu.py re-chunks config 2 into 1776-row chunks,
// tests/multi_gpu_check.py shards 1152 rows over two ranks, both demand bit-level agreement).
bool splittable(const GemmArgs& g) {
  return g.allow_splitk && g.splitk_ws != nullptr && g.stats == nullptr && g.batch == 1 && g.groups == 0 &&
         g.K / kBlockK >= 32;
}

// Row stride of the split-K partials: whole float4 groups for the reduction.
int splitk_ld(int N) { return (N + 7) / 8 * 8; }

// Number of k-slices of a splittable GEMM with `tiles` output tiles (1: no split): up to one work
// item per SM, at most 8, at least 4 k-blocks each, and as many as the workspace holds.
int split_k_factor(const GemmArgs& g, int tiles) {
  const int sms = num_sms();
  if (tiles * 2 > sms) return 1;
  int S = sms / tiles;
  if (S > 8) S = 8;
  if (S > g.K / kBlockK / 4) S = g.K / kBlockK / 4;
  while (S > 1 && (size_t)S * g.M * splitk_ld(g.N) * sizeof(float) > g.splitk_ws_bytes) --S;
  return S;
}

int launch_split_k(const TcParams& p, int bn, int S, const GemmArgs& g, cudaStream_t stream) {
  const int ldw = splitk_ld(g.N);
  TcParams q = p;  // first pass: raw partial sums
  q.split_k = S;
  q.split_stride = (long long)g.M * ldw;
  q.bias = nullptr; q.residual = nullptr; q.act = 0; q.out_planes = nullptr; q.stats = nullptr;
  q.out_f32 = g.splitk_ws; q.ldo = ldw;
  TAPIR_RETURN_IF(launch_gemm(bn, false, q, g, stream));
  const long long total = (long long)g.M * ((g.N + 3) / 4);
  long long blocks = (total + 255) / 256;
  if (blocks > (long long)num_sms() * 8) blocks = (long long)num_sms() * 8;
  splitk_reduce_kernel<<<(unsigned)blocks, 256, 0, stream>>>(g.splitk_ws, S, q.split_stride, ldw, p);
  count_launch();
  TAPIR_LAUNCH_CHECK("splitk_reduce_kernel");
  return kOk;
}

// *v = -1 if the variable `name` is not set, 0 if it is `v0`, 1 if it is `v1`; any other value is
// an error.
int read_switch(const char* name, const char* v0, const char* v1, int* v) {
  *v = -1;
  const char* e = getenv(name);
  if (e == nullptr) return kOk;
  TAPIR_CHECK_ARG(strcmp(e, v0) == 0 || strcmp(e, v1) == 0, "%s='%s': expected %s or %s", name, e, v0, v1);
  *v = strcmp(e, v0) == 0 ? 0 : 1;
  return kOk;
}

}  // namespace

// The one reader of the switches; the rule they follow is stated with GemmSwitches (gemm.cuh).
int read_gemm_switches(GemmSwitches* sw) {
  *sw = GemmSwitches();
  int v;
  TAPIR_RETURN_IF(read_switch("TAPIR_B200_GEMM", "tc", "simt", &v));
  sw->simt = v == 1;
  TAPIR_RETURN_IF(read_switch("TAPIR_B200_BLOCK_N", "64", "128", &v));
  sw->block_n = v < 0 ? 0 : v == 0 ? 64 : 128;
  TAPIR_RETURN_IF(read_switch("TAPIR_B200_GEMM_SCHEDULE", "coop", "pingpong", &v));
  sw->schedule = v + 1;
  TAPIR_RETURN_IF(read_switch("TAPIR_B200_CONV_HALO", "0", "1", &v));
  sw->halo = v != 0;
  return kOk;
}

int validate_gemm_args(const GemmArgs& g) {
  TAPIR_CHECK_ARG(g.planes >= 1 && g.planes <= 3, "gemm: planes must be 1..3 (got %d)", g.planes);
  TAPIR_CHECK_ARG(g.M > 0 && g.N > 0 && g.K > 0, "gemm: empty problem M=%d N=%d K=%d", g.M, g.N, g.K);
  TAPIR_CHECK_ARG(g.K % kBlockK == 0, "gemm: K=%d must be a multiple of 64 (pad with zeros)", g.K);
  TAPIR_CHECK_ARG(g.a != nullptr && g.b != nullptr, "gemm: null operand");
  TAPIR_CHECK_ARG((reinterpret_cast<uintptr_t>(g.a) & 15) == 0 && (reinterpret_cast<uintptr_t>(g.b) & 15) == 0,
                  "gemm: operands must be 16-byte aligned");
  TAPIR_CHECK_ARG(g.ldb >= g.K && g.ldb % 8 == 0, "gemm: ldb=%d must be >= K and a multiple of 8", g.ldb);
  TAPIR_CHECK_ARG(g.b_plane_stride % 8 == 0 && g.a_plane_stride % 8 == 0, "gemm: plane strides must be multiples of 8 elements");
  if (g.mode == kGemmConv3x3) {
    TAPIR_CHECK_ARG(g.C % kBlockK == 0 && g.K == 9 * g.C, "gemm(conv): C=%d must be a multiple of 64 and K=9*C", g.C);
    TAPIR_CHECK_ARG(g.frames > 0 && g.H > 0 && g.W > 0 && (long long)g.frames * g.H * g.W == g.M,
                    "gemm(conv): M must equal frames*H*W");
  } else {
    TAPIR_CHECK_ARG(g.mode == kGemmPlain, "gemm: unknown mode %d", g.mode);
    TAPIR_CHECK_ARG(g.lda >= g.K && g.lda % 8 == 0, "gemm: lda=%d must be >= K and a multiple of 8", g.lda);
  }
  TAPIR_CHECK_ARG(g.out_f32 != nullptr || g.out_planes != nullptr, "gemm: no output");
  if (g.out_planes != nullptr)
    TAPIR_CHECK_ARG(g.out_P >= 1 && g.out_P <= 3 && g.ldp >= g.N, "gemm: bad plane output (out_P=%d ldp=%d)", g.out_P, g.ldp);
  if (g.out_f32 != nullptr) TAPIR_CHECK_ARG(g.ldo >= g.N, "gemm: ldo=%d < N=%d", g.ldo, g.N);
  if (g.residual != nullptr) TAPIR_CHECK_ARG(g.ldr >= g.N, "gemm: ldr=%d < N=%d", g.ldr, g.N);
  TAPIR_CHECK_ARG(g.batch >= 1 && g.batch <= 65535, "gemm: batch=%d must be 1..65535", g.batch);
  if (g.batch > 1) {
    TAPIR_CHECK_ARG(g.mode == kGemmPlain && g.out_f32 != nullptr && g.out_planes == nullptr &&
                        g.residual == nullptr && g.stats == nullptr,
                    "gemm: a batched GEMM is plain mode with an fp32 output and no residual or statistics");
    TAPIR_CHECK_ARG(g.a_batch_rows >= 0 && g.b_batch_rows >= 0 && g.out_batch_stride >= 0,
                    "gemm: negative batch stride");
    const long long arows = g.a_batch_rows > 0 ? g.a_batch_rows : g.M;
    const long long brows = g.b_batch_rows > 0 ? g.b_batch_rows : g.N;
    TAPIR_CHECK_ARG(arows >= g.M && brows >= g.N && arows * g.batch < (1ll << 31) && brows * g.batch < (1ll << 31),
                    "gemm: batch strides out of range");
  }
  if (g.groups != 0) {
    TAPIR_CHECK_ARG(g.groups >= 1 && g.groups <= kGemmMaxGroups && g.batch == 1,
                    "gemm: groups=%d must be 1..%d, with batch 1", g.groups, kGemmMaxGroups);
    TAPIR_CHECK_ARG(g.mode == kGemmPlain && g.out_f32 != nullptr && g.out_planes == nullptr &&
                        g.residual == nullptr && g.stats == nullptr,
                    "gemm: a grouped GEMM is plain mode with an fp32 output and no residual or statistics");
    TAPIR_CHECK_ARG(g.b_batch_rows >= 0 && (long long)(g.groups - 1) * (g.b_batch_rows > 0 ? g.b_batch_rows : g.N) +
                                               g.N < (1ll << 31),
                    "gemm: group B rows out of range");
    TAPIR_CHECK_ARG(g.group_row0[0] == 0 && g.group_row0[g.groups] == g.M, "gemm: group rows must cover [0, M)");
    for (int i = 0; i < g.groups; ++i)
      TAPIR_CHECK_ARG(g.group_row0[i + 1] > g.group_row0[i], "gemm: group %d has no rows", i);
  }
  if (g.stats != nullptr) {
    TAPIR_CHECK_ARG(g.out_planes == nullptr, "gemm: fused statistics need an fp32-only output");
    if (g.mode == kGemmPlain)
      TAPIR_CHECK_ARG(g.rows_per_frame > 0 && g.rows_per_frame % kBlockM == 0 && g.M % g.rows_per_frame == 0,
                      "gemm: fused statistics need rows_per_frame %% 128 == 0 (got %d)", g.rows_per_frame);
  }
  return kOk;
}

int gemm_tc(const GemmArgs& g, const GemmSwitches& sw, cudaStream_t stream) {
  TAPIR_RETURN_IF(validate_gemm_args(g));
  TcParams p;
  TAPIR_RETURN_IF(common_params(g, &p));
  if (use_halo(g, sw)) return launch_halo(p, g, sw, stream);
  const bool split = splittable(g);
  const int bn = pick_block_n(p.num_m_tiles, g.N, split, sw);
  p.num_n_tiles = ceil_div(g.N, bn);
  const int b_problems = g.groups > 0 ? g.groups : g.batch;
  TAPIR_RETURN_IF(encode_rows_map(&p.tmB, g.b, g.K, (b_problems - 1) * p.b_batch_rows + g.N, g.ldb,
                                  g.b_plane_stride, g.planes, bn, "B"));
  const int tiles = p.num_m_tiles * p.num_n_tiles;
  const int S = split ? split_k_factor(g, tiles) : 1;
  if (S > 1) return launch_split_k(p, bn, S, g, stream);
  const bool pingpong = pick_pingpong(tiles, p.num_k_blocks, g.planes, g.batch > 1 || g.groups > 0, sw);
  TAPIR_RETURN_IF(plane_store_params(g, pingpong, &p));
  return launch_gemm(bn, pingpong, p, g, stream);
}

}  // namespace tapir
