// SIMT fp32 implementation of the GemmArgs contract (gemm.cuh).  Not the product path: it is
// the on-device cross-check for the wgmma kernel (tests/test_gemm_gpu.py) and a bring-up
// switch (TAPIR_B200_GEMM=simt).  It reconstructs a = sum_i A_i, b = sum_j B_j in fp32 and
// runs a shared-memory tiled fp32 GEMM; versus the tensor-core path it additionally contains
// the dropped (i + j >= P) cross terms, i.e. it differs by <= 2^-16 relative for P=2.
#include <algorithm>

#include "gemm.cuh"

namespace tapir {

namespace {

constexpr int TM = 64, TN = 64, TK = 16;

struct SimtParams {
  GemmArgs g;
  long long a_plane, b_plane;
  long long a_batch_rows, b_batch_rows, out_batch_stride;  // batch or group = blockIdx.z
};

// Rows of problem blockIdx.z (a batch or a group) and its first A and output row.
__device__ __forceinline__ int problem_rows(const GemmArgs& g) {
  return g.groups > 0 ? g.group_row0[blockIdx.z + 1] - g.group_row0[blockIdx.z] : g.M;
}
__device__ __forceinline__ long long problem_row0(const SimtParams& p) {
  return p.g.groups > 0 ? p.g.group_row0[blockIdx.z] : (long long)blockIdx.z * p.a_batch_rows;
}

__device__ __forceinline__ float load_a(const SimtParams& p, int m, int k) {
  const GemmArgs& g = p.g;
  if (m >= problem_rows(g)) return 0.f;
  long long off;
  if (g.mode == kGemmConv3x3) {
    const int tap = k / g.C, c = k - tap * g.C;
    const int ky = tap / 3, kx = tap - ky * 3;
    const int hw = g.H * g.W;
    const int f = m / hw, r = m - f * hw;
    const int y = r / g.W + ky - 1, x = r % g.W + kx - 1;
    if (y < 0 || y >= g.H || x < 0 || x >= g.W) return 0.f;
    off = (((long long)f * g.H + y) * g.W + x) * g.C + c;
  } else {
    off = (problem_row0(p) + m) * g.lda + k;
  }
  float v = 0.f;
  for (int i = 0; i < g.planes; ++i) v += __bfloat162float(g.a[i * p.a_plane + off]);
  return v;
}

__device__ __forceinline__ float load_b(const SimtParams& p, int n, int k) {
  const GemmArgs& g = p.g;
  if (n >= g.N) return 0.f;
  const long long off = ((long long)blockIdx.z * p.b_batch_rows + n) * g.ldb + k;
  float v = 0.f;
  for (int i = 0; i < g.planes; ++i) v += __bfloat162float(g.b[i * p.b_plane + off]);
  return v;
}

__global__ void __launch_bounds__(256) gemm_simt_kernel(const __grid_constant__ SimtParams p) {
  __shared__ float As[TK][TM + 4];
  __shared__ float Bs[TK][TN + 4];
  const GemmArgs& g = p.g;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int m0 = blockIdx.x * TM, n0 = blockIdx.y * TN;
  const int rows = problem_rows(g);
  float* out_f32 = g.out_f32 == nullptr ? nullptr
                   : g.groups > 0       ? g.out_f32 + problem_row0(p) * g.ldo
                                        : g.out_f32 + blockIdx.z * p.out_batch_stride;
  float acc[4][4] = {};
  for (int k0 = 0; k0 < g.K; k0 += TK) {
    for (int e = threadIdx.x; e < TM * TK; e += 256) {
      const int kk = e & (TK - 1), mm = e / TK;
      As[kk][mm] = load_a(p, m0 + mm, k0 + kk);
      Bs[kk][mm] = load_b(p, n0 + mm, k0 + kk);
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < TK; ++kk) {
      float a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = As[kk][ty * 4 + i];
#pragma unroll
      for (int j = 0; j < 4; ++j) b[j] = Bs[kk][tx * 4 + j];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
  for (int i = 0; i < 4; ++i) {
    const long long m = m0 + ty * 4 + i;
    if (m >= rows) continue;
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx * 4 + j;
      if (n >= g.N) continue;
      float v = acc[i][j];
      if (g.bias != nullptr) v += g.bias[n];
      if (g.act == 1) v = gelu_tanh(v);
      if (g.residual != nullptr) v += g.residual[m * g.ldr + n];
      if (out_f32 != nullptr) out_f32[m * g.ldo + n] = v;
      if (g.stats != nullptr) {
        const long long rpf = (g.mode == kGemmConv3x3) ? (long long)g.H * g.W : (g.rows_per_frame > 0 ? g.rows_per_frame : g.M);
        double* dst = g.stats + ((m / rpf) * g.N + n) * 2;
        atomicAdd(dst, (double)v);
        atomicAdd(dst + 1, (double)v * v);
      }
      if (g.out_planes != nullptr) {
        float r = v;
        for (int q = 0; q < g.out_P; ++q) {
          __nv_bfloat16 h = __float2bfloat16_rn(r);
          r -= __bfloat162float(h);
          g.out_planes[q * g.out_plane_stride + m * g.ldp + n] = h;
        }
      }
    }
  }
}

}  // namespace

int gemm_simt(const GemmArgs& g, cudaStream_t stream) {
  TAPIR_RETURN_IF(validate_gemm_args(g));
  SimtParams p;
  p.g = g;
  p.a_batch_rows = g.a_batch_rows > 0 ? g.a_batch_rows : g.M;
  p.b_batch_rows = g.b_batch_rows > 0 ? g.b_batch_rows : g.N;
  p.out_batch_stride = g.out_batch_stride > 0 ? g.out_batch_stride : (long long)g.M * g.ldo;
  // default plane strides span every batch's rows
  if (g.mode == kGemmConv3x3) {
    p.a_plane = g.a_plane_stride > 0 ? g.a_plane_stride : (long long)g.M * g.C;
  } else {
    p.a_plane = g.a_plane_stride > 0 ? g.a_plane_stride : ((g.batch - 1) * p.a_batch_rows + g.M) * g.lda;
  }
  p.b_plane = g.b_plane_stride > 0 ? g.b_plane_stride
                                   : ((std::max(g.batch, g.groups) - 1) * p.b_batch_rows + g.N) * g.ldb;
  ProfileScope ps(g.tag ? g.tag : "gemm", stream,
                  2.0 * g.batch * g.M * g.N * (g.k_logical > 0 ? g.k_logical : g.K), 0.0);
  int rows = g.M, problems = g.batch;
  if (g.groups > 0) {
    problems = g.groups;
    rows = 0;
    for (int i = 0; i < g.groups; ++i) rows = std::max(rows, g.group_row0[i + 1] - g.group_row0[i]);
  }
  dim3 grid(ceil_div(rows, TM), ceil_div(g.N, TN), problems);
  gemm_simt_kernel<<<grid, 256, 0, stream>>>(p);
  count_launch();
  TAPIR_LAUNCH_CHECK("gemm_simt_kernel");
  return kOk;
}

int gemm(const GemmArgs& g, cudaStream_t stream) {
  GemmSwitches sw;
  TAPIR_RETURN_IF(read_gemm_switches(&sw));
  return sw.simt ? gemm_simt(g, stream) : gemm_tc(g, sw, stream);
}

}  // namespace tapir
