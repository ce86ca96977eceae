// Shared device/host helpers for the tapir_b200 kernels (sm_90a only).
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <cstdio>
#include <cstring>

namespace tapir {

// ---------------------------------------------------------------------------------------
// error plumbing: every extern "C" entry returns 0 on success; message via tapir_last_error
// ---------------------------------------------------------------------------------------
enum Status : int {
  kOk = 0,
  kBadArgument = 1,
  kUnsupported = 2,
  kCudaError = 3,
  kWorkspaceTooSmall = 4,
};

void set_error(const char* fmt, ...);
int cuda_fail(cudaError_t e, const char* what);

#define TAPIR_CHECK_ARG(cond, ...)                 \
  do {                                             \
    if (!(cond)) {                                 \
      ::tapir::set_error(__VA_ARGS__);             \
      return ::tapir::kBadArgument;                \
    }                                              \
  } while (0)

#define TAPIR_CUDA(expr)                                        \
  do {                                                          \
    cudaError_t _e = (expr);                                    \
    if (_e != cudaSuccess) return ::tapir::cuda_fail(_e, #expr); \
  } while (0)

#define TAPIR_LAUNCH_CHECK(name)                                     \
  do {                                                               \
    cudaError_t _e = cudaGetLastError();                             \
    if (_e != cudaSuccess) return ::tapir::cuda_fail(_e, name);      \
  } while (0)

#define TAPIR_RETURN_IF(expr)        \
  do {                               \
    int _s = (expr);                 \
    if (_s != 0) return _s;          \
  } while (0)

int num_sms();  // of the CURRENT device

// Per-device one-time setup (cudaFuncSetAttribute, scratch allocations): every cache in this
// library is keyed by cudaGetDevice(), so several GPUs can be driven from one process.
constexpr int kMaxDevices = 64;
int current_device();  // cudaGetDevice(), clamped to [0, kMaxDevices)
struct PerDeviceOnce {
  bool done[kMaxDevices] = {};
  // true exactly once per device; call mark() after the setup succeeded
  bool pending() const { return !done[current_device()]; }
  void mark() { done[current_device()] = true; }
};

// counts kernels launched by this library (bench.py reports it as gpu_launches)
extern unsigned long long g_launch_count;
inline void count_launch(int n = 1) { g_launch_count += (unsigned long long)n; }

// Optional per-launch device timing (tapir_profile_*): when enabled, a ProfileScope records a
// CUDA event pair on the launch stream around one kernel launch and books the launch's
// algorithmic FLOPs / bytes under `name`.  bench.py uses it for the roofline object.
extern bool g_profile_on;
struct ProfileScope {
  int slot;
  cudaStream_t stream;
  ProfileScope(const char* name, cudaStream_t s, double flops, double bytes);
  ~ProfileScope();
};

static inline int ceil_div(int a, int b) { return (a + b - 1) / b; }
static inline long long ceil_div_ll(long long a, long long b) { return (a + b - 1) / b; }
static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// ---------------------------------------------------------------------------------------
// device helpers
// ---------------------------------------------------------------------------------------
#ifdef __CUDACC__

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// tanh-approximated GELU, F.gelu(x, approximate='tanh') (nets.py:59,102,160):
//   0.5 x (1 + tanh(k (x + 0.044715 x^3))) == x * sigmoid(2 k (x + 0.044715 x^3))
// evaluated through ex2.approx (|rel err| ~1e-6, far inside the 1e-4 logit budget).
__device__ __forceinline__ float gelu_tanh(float x) {
  // e = exp(-2k(x + c x^3)) = 2^(x * (A + B x^2)),  A = -2k log2(e),  B = A * 0.044715
  const float A = -2.3022081983f;
  const float B = -0.1029432396f;
  const float u = x * fmaf(x * x, B, A);
  float e, r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(u));
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(1.0f + e));  // 1 + e in [1, +inf]: see gelu_tanh2
  return x * r;
}

// Elementwise fp32 pair arithmetic, each half an IEEE round-to-nearest operation (never
// contracted or reassociated).  Hopper has no packed fp32 instructions: two scalar ops each.
__device__ __forceinline__ float2 fma2_rn(float2 a, float2 b, float2 c) {
  return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}
__device__ __forceinline__ float2 mul2_rn(float2 a, float2 b) {
  return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y));
}
__device__ __forceinline__ float2 add2_rn(float2 a, float2 b) {
  return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y));
}

// Two tanh-GELUs on an fp32 pair.  Same formula and rounding as gelu_tanh.
__device__ __forceinline__ float2 gelu_tanh2(float2 x) {
  const float2 A = make_float2(-2.3022081983f, -2.3022081983f);
  const float2 B = make_float2(-0.1029432396f, -0.1029432396f);
  const float2 u = mul2_rn(x, fma2_rn(mul2_rn(x, x), B, A));
  float2 e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e.x) : "f"(u.x));
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e.y) : "f"(u.y));
  const float2 d = add2_rn(e, make_float2(1.0f, 1.0f));
  // d is in [1, +inf]: rcp.approx needs none of div.approx's range handling (which costs an
  // FSETP and two FMULs per division); rcp(+inf) = 0 gives gelu(-large) = -0 like the quotient
  float2 r;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r.x) : "f"(d.x));
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r.y) : "f"(d.y));
  return mul2_rn(x, r);
}

// One step of the bf16 split for two values at once: returns bf16x2(a, b) (a in the low half)
// and replaces a, b by their residuals.  Uses the packed convert (F2FP, full rate) instead of
// two scalar F2F conversions (quarter-rate unit, scoreboard latency).
__device__ __forceinline__ uint32_t bf16x2_split(float& a, float& b) {
  const __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  const uint32_t u = *reinterpret_cast<const uint32_t*>(&h);
  a -= __uint_as_float(u << 16);
  b -= __uint_as_float(u & 0xffff0000u);
  return u;
}

// Split an fp32 value into P bf16 terms: x ~= p0 + p1 (+ p2); each term is the bf16
// rounding of the remaining residual.  P=2 carries ~16 mantissa bits, P=3 all 24.
template <int P>
__device__ __forceinline__ void split_bf16(float x, __nv_bfloat16 (&out)[P]) {
  float r = x;
#pragma unroll
  for (int i = 0; i < P; ++i) {
    out[i] = __float2bfloat16_rn(r);
    r = r - __bfloat162float(out[i]);
  }
}

#endif  // __CUDACC__

}  // namespace tapir
