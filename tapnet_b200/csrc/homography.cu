// Camera homographies from point tracks, as the reference's get_homographies_wrt_frame
// (tapnet/utils/viz_utils.py:301-648), in float64 (DESIGN section 10, row f8).
//
// The frame steps are sequential: each frame's RANSAC targets the canonical points the step before
// it left.  Every step is a fixed launch sequence; every decision (the > 4 gate, the RANSAC stop,
// the no-inlier fallback) is read on the device, so a call never syncs with the host:
//   * sweep frame i:   prep (1 CTA) -> score (<= kScoreCtas CTAs) -> estimate (1 CTA) -> canonical
//   * refinement fr:   refine (1 CTA) -> canonical
//   * reference frame of refinement pass j < last: refine -> canonical (all-err form) -> canonical
// plus one init and one output launch per call.
//
// RANSAC.  Hypothesis k draws 4 ranks among the frame's usable points with Floyd's algorithm over
// SplitMix64 (homography_oracle.hypothesis_ranks), solves the 8 x 9 system's null vector as the
// smallest eigenvector of its 9 x 9 normal matrix (Jacobi in one warp), and counts err < thresh^2
// over all N points.  One warp scores one hypothesis; a CTA scores a block of kHypWarps.  The CTA
// that finishes a block publishes it, and whichever CTA holds the scan lock walks the completed
// prefix of blocks hypothesis by hypothesis exactly as the sequential loop does (a strictly greater
// count replaces the kept one; stop after k once best >= thr[k + 1]).  The lock is only ever tried,
// never waited for: a CTA that finds it taken leaves, and the holder re-checks the next block after
// releasing it, so no CTA waits on another.  Once the scan has stopped, CTAs skip the blocks they
// have not started.
//
// Estimates accumulate the 9 x 9 normal equations per thread over a fixed point assignment and
// reduce them in a fixed order (no atomics), so every result repeats bit for bit.
#include <cuda/atomic>

#include <algorithm>
#include <cmath>

#include "kernels.cuh"

namespace tapir {
namespace {

constexpr int kHypWarps = 8;        // hypotheses per scan block: one per warp of a score CTA
constexpr int kScoreCtas = 32;      // score CTAs: kScoreCtas * kHypWarps hypotheses in flight
constexpr int kSolveThreads = 256;  // the 1-CTA estimate kernels
constexpr int kCanonWarps = 16;     // canonical kernel: 32 points x 16 frame slices per CTA
constexpr int kPrepThreads = 1024;
constexpr int kJacobiSweeps = 16;

enum { kM, kGate, kStopped, kFrontier, kLock, kBest, kBestK, kEvaluated, kStateInts };

using AtomicInt = cuda::atomic_ref<int, cuda::thread_scope_device>;

// Workspace: frame-major float64 copies of the inputs and the loop's state.
struct Ws {
  double* pts;      // [T][N][2] normalised points
  double* tformed;  // [T][N][2] every frame's points in the canonical frame
  double* err;      // [T][N]
  double* canon;    // [N][2]
  double* res;      // [T][9] homographies, unscaled
  double* hcur;     // [9] the homography of the current step
  uint8_t* occ;     // [T][N]
  uint8_t* inval;   // [T][N] occlusion of visited frames; 1 for frames the sweep has not reached
  uint8_t* cbad;    // [N] canonical_invalid
  int* usable;      // [N] the current frame's usable points in index order
  int* counts;      // [N] inlier count of each hypothesis
  int* done;        // [scan blocks]
  int* state;       // [kStateInts]
};

__host__ __device__ int scan_blocks(int N) { return N > 1 ? (N - 1 + kHypWarps - 1) / kHypWarps : 1; }

Ws carve(Arena& a, int T, int N) {
  const size_t tn = (size_t)T * N;
  Ws w;
  w.pts = a.take<double>(tn * 2);
  w.tformed = a.take<double>(tn * 2);
  w.err = a.take<double>(tn);
  w.canon = a.take<double>((size_t)N * 2);
  w.res = a.take<double>((size_t)T * 9);
  w.hcur = a.take<double>(9);
  w.occ = a.take<uint8_t>(tn);
  w.inval = a.take<uint8_t>(tn);
  w.cbad = a.take<uint8_t>(N);
  w.usable = a.take<int>(N);
  w.counts = a.take<int>(N);
  w.done = a.take<int>(scan_blocks(N));
  w.state = a.take<int>(kStateInts);
  return w;
}

__host__ __device__ __forceinline__ uint64_t mix64(uint64_t x) {
  uint64_t z = x + 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

struct Tf {
  double x, y, err;
};

// compute_inliers for one point: H (row-major) applied to (sx, sy, sx * 0 + 1), divided by
// max(1e-12, |w|) * sign(w) with numpy's NaN propagation, err against (tx, ty).  Products and sums
// are rounded one by one in numpy's order.
__device__ __forceinline__ Tf transform(const double* h, double sx, double sy, double tx, double ty) {
  const double one = __dadd_rn(__dmul_rn(sx, 0.0), 1.0);
  double v[3];
#pragma unroll
  for (int r = 0; r < 3; ++r)
    v[r] = __dadd_rn(__dadd_rn(__dmul_rn(h[3 * r], sx), __dmul_rn(h[3 * r + 1], sy)),
                     __dmul_rn(h[3 * r + 2], one));
  const double aw = fabs(v[2]);
  const double m = aw != aw ? aw : (aw > 1e-12 ? aw : 1e-12);
  const double sg = v[2] > 0.0 ? 1.0 : (v[2] < 0.0 ? -1.0 : (v[2] == 0.0 ? 0.0 : v[2]));
  const double d = __dmul_rn(m, sg);
  Tf o;
  o.x = __ddiv_rn(v[0], d);
  o.y = __ddiv_rn(v[1], d);
  const double dx = __dsub_rn(tx, o.x), dy = __dsub_rn(ty, o.y);
  o.err = __dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy));
  return o;
}

// The two rows estimate_homography builds from one correspondence (targ = H src), times mask.
__device__ __forceinline__ void system_rows(double tx, double ty, double sx, double sy, double m,
                                            double (&r1)[9], double (&r2)[9]) {
  const double a[9] = {sx, sy, 1.0, 0.0, 0.0, 0.0, -tx * sx, -tx * sy, -tx};
  const double b[9] = {0.0, 0.0, 0.0, sx, sy, 1.0, -ty * sx, -ty * sy, -ty};
#pragma unroll
  for (int i = 0; i < 9; ++i) {
    r1[i] = a[i] * m;
    r2[i] = b[i] * m;
  }
}

// Upper triangle of the 9 x 9 normal matrix, row by row: 45 entries.
__device__ __forceinline__ void accumulate_rows(const double (&r1)[9], const double (&r2)[9],
                                                double (&acc)[45]) {
  int e = 0;
#pragma unroll
  for (int i = 0; i < 9; ++i)
#pragma unroll
    for (int j = i; j < 9; ++j, ++e) acc[e] += r1[i] * r1[j] + r2[i] * r2[j];
}

// Shared scratch of one warp's eigen-solve.
struct Solve {
  double M[81], V[81], M2[81], V2[81];
  double d[9], o[9];
  int partner[9];
  double h[9];
  double pt[4][4];  // a hypothesis' 4 correspondences (tx, ty, sx, sy)
};

// The unit eigenvector of the smallest eigenvalue of the symmetric 9 x 9 s.M (full, row-major)
// into s.h, by cyclic Jacobi in one warp: each round applies 4 disjoint rotations (the circle
// schedule over 9 indices), each lane updating up to 3 entries of M and V.  Ties go to the larger
// index, so the zero matrix gives e9, as LAPACK's SVD does.  All 32 lanes call it.
__device__ void smallest_eigvec(Solve& s) {
  const int lane = threadIdx.x & 31;
  for (int e = lane; e < 81; e += 32) s.V[e] = (e / 9 == e % 9) ? 1.0 : 0.0;
  __syncwarp();
  for (int sweep = 0; sweep < kJacobiSweeps; ++sweep) {
    bool rotated = false;
    for (int r = 0; r < 9; ++r) {
      if (lane < 9) {
        s.d[lane] = 1.0;
        s.o[lane] = 0.0;
        s.partner[lane] = lane;
      }
      __syncwarp();
      bool mine = false;
      if (lane < 4) {
        const int a = (r + lane + 1) % 9, b = (r + 8 - lane) % 9;
        const int p = a < b ? a : b, q = a < b ? b : a;
        const double app = s.M[p * 9 + p], aqq = s.M[q * 9 + q], apq = s.M[p * 9 + q];
        double c = 1.0, sn = 0.0;
        if (fabs(apq) > 2e-16 * sqrt(fabs(app * aqq)) && fabs(apq) > 1e-300) {
          const double tau = (aqq - app) / (2.0 * apq);
          const double t = (tau >= 0.0 ? 1.0 : -1.0) / (fabs(tau) + sqrt(1.0 + tau * tau));
          c = 1.0 / sqrt(1.0 + t * t);
          sn = t * c;
          mine = true;
        }
        s.d[p] = c;
        s.d[q] = c;
        s.o[p] = -sn;
        s.o[q] = sn;
        s.partner[p] = q;
        s.partner[q] = p;
      }
      rotated |= __any_sync(0xffffffffu, mine);
      __syncwarp();
      for (int e = lane; e < 81; e += 32) {
        const int i = e / 9, j = e % 9, ip = s.partner[i], jp = s.partner[j];
        const double di = s.d[i], oi = s.o[i], dj = s.d[j], oj = s.o[j];
        double v = di * dj * s.M[i * 9 + j] + di * oj * s.M[i * 9 + jp] + oi * dj * s.M[ip * 9 + j] +
                   oi * oj * s.M[ip * 9 + jp];
        if (ip == j && i != j) v = 0.0;  // the rotated pair's entry is zero by construction
        s.M2[e] = v;
        s.V2[e] = s.V[i * 9 + j] * dj + s.V[i * 9 + jp] * oj;
      }
      __syncwarp();
      for (int e = lane; e < 81; e += 32) {
        s.M[e] = s.M2[e];
        s.V[e] = s.V2[e];
      }
      __syncwarp();
    }
    if (!rotated) break;
  }
  int best = 0;
  for (int j = 1; j < 9; ++j)
    if (s.M[j * 9 + j] <= s.M[best * 9 + best]) best = j;
  if (lane < 9) s.h[lane] = s.V[lane * 9 + best];
  __syncwarp();
}

// Hypothesis k of frame i into s.h (all lanes of one warp; the frame has m >= 5 usable points).
__device__ void hypothesis(const Ws& w, int N, int i, int k, Solve& s) {
  const int lane = threadIdx.x & 31;
  if (lane == 0) {
    const int m = w.state[kM];
    const uint64_t seed = mix64(0);
    int rank[4];
    for (int d = 0; d < 4; ++d) {
      const uint64_t j = (uint64_t)(m - 4 + d);
      uint64_t r = ((mix64(seed ^ (((uint64_t)k << 2) | (uint64_t)d)) >> 32) * (j + 1)) >> 32;
      for (int e = 0; e < d; ++e)
        if ((uint64_t)rank[e] == r) r = j;
      rank[d] = (int)r;
    }
    for (int d = 0; d < 4; ++d) {
      const long long n = w.usable[rank[d]];
      s.pt[d][0] = w.canon[2 * n];
      s.pt[d][1] = w.canon[2 * n + 1];
      s.pt[d][2] = w.pts[((long long)i * N + n) * 2];
      s.pt[d][3] = w.pts[((long long)i * N + n) * 2 + 1];
    }
  }
  __syncwarp();
  for (int e = lane; e < 81; e += 32) {
    const int a = e / 9, b = e % 9;
    double acc = 0.0;
    for (int half = 0; half < 2; ++half)  // the 4 x-rows, then the 4 y-rows
      for (int d = 0; d < 4; ++d) {
        double r1[9], r2[9];
        system_rows(s.pt[d][0], s.pt[d][1], s.pt[d][2], s.pt[d][3], 1.0, r1, r2);
        const double* r = half ? r2 : r1;
        acc += r[a] * r[b];
      }
    s.M[e] = acc;
  }
  __syncwarp();
  smallest_eigvec(s);
  // One correction step on the system's own rows (corrected semi-normal equations): with A the
  // 8 x 9 system and M = A^T A = V diag(lambda) V^T from Jacobi, h -= sum_{i != null} v_i (v_i^T
  // A^T A h) / lambda_i.  Forming M squares the condition number; the step brings the null vector
  // back to the accuracy of an SVD of A (eps kappa(A)), so inlier counts follow the reference's.
  double* r = s.M2;       // [8] residual A h
  double* g = s.M2 + 8;   // [9] A^T r
  double* hn = s.M2 + 17; // [9] corrected h
  int nul = 0;
  for (int j = 1; j < 9; ++j)
    if (s.M[j * 9 + j] <= s.M[nul * 9 + nul]) nul = j;
  if (lane < 8) {
    double r1[9], r2[9];
    system_rows(s.pt[lane & 3][0], s.pt[lane & 3][1], s.pt[lane & 3][2], s.pt[lane & 3][3], 1.0, r1, r2);
    double acc = 0.0;
    for (int k = 0; k < 9; ++k) acc += (lane < 4 ? r1[k] : r2[k]) * s.h[k];
    r[lane] = acc;
  }
  __syncwarp();
  if (lane < 9) {
    double acc = 0.0;
    for (int d = 0; d < 4; ++d) {
      double r1[9], r2[9];
      system_rows(s.pt[d][0], s.pt[d][1], s.pt[d][2], s.pt[d][3], 1.0, r1, r2);
      acc += r1[lane] * r[d] + r2[lane] * r[4 + d];
    }
    g[lane] = acc;
  }
  __syncwarp();
  if (lane < 9) {
    double delta = 0.0;
    for (int i = 0; i < 9; ++i) {
      const double lam = s.M[i * 9 + i];
      if (i == nul || !(lam > 0.0)) continue;
      double c = 0.0;
      for (int k = 0; k < 9; ++k) c += s.V[k * 9 + i] * g[k];
      delta += s.V[lane * 9 + i] * (c / lam);
    }
    hn[lane] = s.h[lane] - delta;
  }
  __syncwarp();
  double norm = 0.0;
  for (int k = 0; k < 9; ++k) norm += hn[k] * hn[k];
  norm = sqrt(norm);
  if (lane < 9) s.h[lane] = hn[lane] / norm;
  __syncwarp();
}

// Fixed-order block reduction of per-thread acc[45] into s.M (full symmetric), then the smallest
// eigenvector into s.h by warp 0.  red: [kSolveThreads / 32][45] shared doubles.
__device__ void solve_normal(double (&acc)[45], double* red, Solve& s) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int e = 0; e < 45; ++e) {
    double v = acc[e];
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
    if (lane == 0) red[warp * 45 + e] = v;
  }
  __syncthreads();
  if (warp == 0) {
    for (int e = lane; e < 45; e += 32) {
      double v = 0.0;
      for (int x = 0; x < kSolveThreads / 32; ++x) v += red[x * 45 + e];
      int i = 0, rem = e;
      while (rem >= 9 - i) {
        rem -= 9 - i;
        ++i;
      }
      const int j = i + rem;
      s.M[i * 9 + j] = v;
      s.M[j * 9 + i] = v;
    }
    __syncwarp();
    smallest_eigvec(s);
  }
  __syncthreads();
}

// ---------------------------------------------------------------------------------------------
__global__ void init_kernel(tapir_homography_args a, Ws w) {
  const int T = a.T, N = a.N;
  const long long tn = (long long)T * N;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < tn;
       idx += (long long)gridDim.x * blockDim.x) {
    const int t = (int)(idx / N), n = (int)(idx % N);
    const long long src = (long long)n * T + t;
    double x, y;
    if (a.tracks_fp64) {
      x = static_cast<const double*>(a.tracks)[2 * src];
      y = static_cast<const double*>(a.tracks)[2 * src + 1];
    } else {
      x = static_cast<const float*>(a.tracks)[2 * src];
      y = static_cast<const float*>(a.tracks)[2 * src + 1];
    }
    x = __ddiv_rn(x, a.width);
    y = __ddiv_rn(y, a.height);
    const uint8_t o = a.occluded[src] != 0;
    const bool ref = t == a.reference_frame;
    w.pts[2 * idx] = x;
    w.pts[2 * idx + 1] = y;
    w.occ[idx] = o;
    w.inval[idx] = ref ? o : 1;
    w.tformed[2 * idx] = ref ? x : 0.0;
    w.tformed[2 * idx + 1] = ref ? y : 0.0;
    w.err[idx] = 0.0;
    if (ref) {
      w.canon[2 * n] = x;
      w.canon[2 * n + 1] = y;
      w.cbad[n] = o;
    }
  }
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < 9ll * T;
       idx += (long long)gridDim.x * blockDim.x) {
    const int e = (int)(idx % 9);
    w.res[idx] = (idx / 9 == a.reference_frame && e % 4 == 0) ? 1.0 : 0.0;
    if (a.ransac_stats != nullptr && e < 2) a.ransac_stats[2 * (idx / 9) + e] = 0;
  }
}

// Usable points of frame i (visible there and canonical-valid) in index order, the > 4 gate, and
// a fresh scan state.
__global__ void __launch_bounds__(kPrepThreads) prep_kernel(Ws w, int N, int i) {
  __shared__ int warp_total[kPrepThreads / 32];
  __shared__ int base;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) base = 0;
  __syncthreads();
  for (int n0 = 0; n0 < N; n0 += kPrepThreads) {
    const int n = n0 + threadIdx.x;
    const bool use = n < N && !w.cbad[n] && !w.occ[(long long)i * N + n];
    const unsigned ballot = __ballot_sync(0xffffffffu, use);
    if (lane == 0) warp_total[warp] = __popc(ballot);
    __syncthreads();
    int before = base;
    for (int x = 0; x < warp; ++x) before += warp_total[x];
    if (use) w.usable[before + __popc(ballot & ((1u << lane) - 1u))] = n;
    __syncthreads();
    if (threadIdx.x == 0)
      for (int x = 0; x < kPrepThreads / 32; ++x) base += warp_total[x];
    __syncthreads();
  }
  const int nb = scan_blocks(N);
  for (int b = threadIdx.x; b < nb; b += kPrepThreads) w.done[b] = 0;
  if (threadIdx.x == 0) {
    w.state[kM] = base;
    w.state[kGate] = base > 4;
    w.state[kStopped] = 0;
    w.state[kFrontier] = 0;
    w.state[kLock] = 0;
    w.state[kBest] = 0;
    w.state[kBestK] = -1;
    w.state[kEvaluated] = 0;
  }
}

// Walk the completed prefix of scan blocks as the sequential loop does (one thread).
__device__ void advance_scan(const Ws& w, const double* thr, int N, int nb) {
  AtomicInt lock(w.state[kLock]);
  while (true) {
    int expected = 0;
    if (!lock.compare_exchange_strong(expected, 1, cuda::memory_order_acquire)) return;
    int f = AtomicInt(w.state[kFrontier]).load(cuda::memory_order_relaxed);
    int stopped = AtomicInt(w.state[kStopped]).load(cuda::memory_order_relaxed);
    int best = AtomicInt(w.state[kBest]).load(cuda::memory_order_relaxed);
    int best_k = AtomicInt(w.state[kBestK]).load(cuda::memory_order_relaxed);
    int evaluated = AtomicInt(w.state[kEvaluated]).load(cuda::memory_order_relaxed);
    while (!stopped && f < nb && AtomicInt(w.done[f]).load(cuda::memory_order_acquire)) {
      for (int x = 0; x < kHypWarps && !stopped; ++x) {
        const int k = f * kHypWarps + x;
        if (k > N - 2) break;
        const int c = AtomicInt(w.counts[k]).load(cuda::memory_order_relaxed);
        if (c > best) {
          best = c;
          best_k = k;
        }
        evaluated = k + 1;
        if ((double)best >= thr[k + 1]) stopped = 1;
      }
      ++f;
    }
    AtomicInt(w.state[kFrontier]).store(f, cuda::memory_order_relaxed);
    AtomicInt(w.state[kBest]).store(best, cuda::memory_order_relaxed);
    AtomicInt(w.state[kBestK]).store(best_k, cuda::memory_order_relaxed);
    AtomicInt(w.state[kEvaluated]).store(evaluated, cuda::memory_order_relaxed);
    AtomicInt(w.state[kStopped]).store(stopped, cuda::memory_order_relaxed);
    lock.store(0, cuda::memory_order_release);
    // a block published while the lock was held may have found it taken: look again
    cuda::atomic_thread_fence(cuda::memory_order_seq_cst, cuda::thread_scope_device);
    if (stopped || f >= nb || !AtomicInt(w.done[f]).load(cuda::memory_order_acquire)) return;
  }
}

__global__ void __launch_bounds__(kHypWarps * 32) score_kernel(Ws w, const double* thr, int N, int i,
                                                                double t2) {
  __shared__ Solve solve[kHypWarps];
  __shared__ int skip;
  if (!w.state[kGate]) return;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int nb = scan_blocks(N);
  const double* src = w.pts + (long long)i * N * 2;
  for (int b = blockIdx.x; b < nb; b += gridDim.x) {
    if (threadIdx.x == 0) skip = AtomicInt(w.state[kStopped]).load(cuda::memory_order_relaxed);
    __syncthreads();
    if (skip) return;
    const int k = b * kHypWarps + warp;
    if (k <= N - 2) {
      Solve& s = solve[warp];
      hypothesis(w, N, i, k, s);
      int count = 0;
      for (int n = lane; n < N; n += 32)
        count += transform(s.h, src[2 * n], src[2 * n + 1], w.canon[2 * n], w.canon[2 * n + 1]).err < t2;
      count = __reduce_add_sync(0xffffffffu, count);
      if (lane == 0) AtomicInt(w.counts[k]).store(count, cuda::memory_order_relaxed);
    }
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
      AtomicInt(w.done[b]).store(1, cuda::memory_order_release);
      cuda::atomic_thread_fence(cuda::memory_order_seq_cst, cuda::thread_scope_device);
      advance_scan(w, thr, N, nb);
    }
  }
}

// Normal equations of frame `fr` against the canonical points, with mask[n] given by `keep`.
template <typename Keep>
__device__ void frame_normal(const Ws& w, int N, int fr, Keep keep, double (&acc)[45]) {
#pragma unroll
  for (int e = 0; e < 45; ++e) acc[e] = 0.0;
  const double* src = w.pts + (long long)fr * N * 2;
  for (int n = threadIdx.x; n < N; n += kSolveThreads) {
    const double tx = w.canon[2 * n], ty = w.canon[2 * n + 1], sx = src[2 * n], sy = src[2 * n + 1];
    double r1[9], r2[9];
    system_rows(tx, ty, sx, sy, keep(n, sx, sy, tx, ty) ? 1.0 : 0.0, r1, r2);
    accumulate_rows(r1, r2, acc);
  }
}

// Sweep frame i: the final RANSAC estimate from the best hypothesis' inliers (identity when the
// gate failed), into res[i] and hcur.
__global__ void __launch_bounds__(kSolveThreads) estimate_kernel(tapir_homography_args a, Ws w, int i,
                                                                  double t2) {
  __shared__ Solve s;
  __shared__ double red[kSolveThreads / 32 * 45];
  const int N = a.N;
  const bool gate = w.state[kGate];
  if (gate) {
    const int best_k = w.state[kBestK];
    if (threadIdx.x < 32) {
      if (best_k >= 0) {
        hypothesis(w, N, i, best_k, s);
      } else if (threadIdx.x < 9) {
        s.h[threadIdx.x] = 0.0;  // no hypothesis had an inlier: the zero matrix is kept
      }
    }
    __syncthreads();
    double acc[45];
    frame_normal(w, N, i, [&](int, double sx, double sy, double tx, double ty) {
      return transform(s.h, sx, sy, tx, ty).err < t2;
    }, acc);
    __syncthreads();
    solve_normal(acc, red, s);
  } else if (threadIdx.x < 9) {
    s.h[threadIdx.x] = threadIdx.x % 4 == 0 ? 1.0 : 0.0;
  }
  __syncthreads();
  if (threadIdx.x < 9) {
    w.res[i * 9 + threadIdx.x] = s.h[threadIdx.x];
    w.hcur[threadIdx.x] = s.h[threadIdx.x];
  }
  if (threadIdx.x == 0 && a.ransac_stats != nullptr) {
    a.ransac_stats[2 * i] = gate ? w.state[kEvaluated] : 0;
    a.ransac_stats[2 * i + 1] = gate ? w.state[kBest] : 0;
  }
}

// Refinement of frame fr: re-estimate from the points within thresh of the canonical points.  The
// reference frame's branch (pass j < last) pre-multiplies every homography by the inverse,
// rewrites tformed[fr] with the last frame's points, and keeps the identity.
__global__ void __launch_bounds__(kSolveThreads) refine_kernel(tapir_homography_args a, Ws w, int fr,
                                                                int branch, double t2) {
  __shared__ Solve s;
  __shared__ double red[kSolveThreads / 32 * 45];
  __shared__ double hfr[9], hinv[9];
  const int N = a.N, T = a.T;
  if (threadIdx.x < 9) hfr[threadIdx.x] = w.res[fr * 9 + threadIdx.x];
  __syncthreads();
  const uint8_t* occ = w.occ + (long long)fr * N;
  double acc[45];
  frame_normal(w, N, fr, [&](int n, double sx, double sy, double tx, double ty) {
    const double e = transform(hfr, sx, sy, tx, ty).err;
    return !(w.cbad[n] || e > t2 || occ[n]);
  }, acc);
  solve_normal(acc, red, s);
  if (branch) {
    if (threadIdx.x == 0) {
      const double* m = s.h;
      const double c00 = m[4] * m[8] - m[5] * m[7], c01 = m[5] * m[6] - m[3] * m[8],
                   c02 = m[3] * m[7] - m[4] * m[6];
      const double det = m[0] * c00 + m[1] * c01 + m[2] * c02;
      hinv[0] = c00 / det;
      hinv[1] = (m[2] * m[7] - m[1] * m[8]) / det;
      hinv[2] = (m[1] * m[5] - m[2] * m[4]) / det;
      hinv[3] = c01 / det;
      hinv[4] = (m[0] * m[8] - m[2] * m[6]) / det;
      hinv[5] = (m[2] * m[3] - m[0] * m[5]) / det;
      hinv[6] = c02 / det;
      hinv[7] = (m[1] * m[6] - m[0] * m[7]) / det;
      hinv[8] = (m[0] * m[4] - m[1] * m[3]) / det;
    }
    __syncthreads();
    for (int t = threadIdx.x; t < T; t += kSolveThreads) {
      double r[9], o[9];
      for (int e = 0; e < 9; ++e) r[e] = w.res[t * 9 + e];
      for (int x = 0; x < 3; ++x)
        for (int y = 0; y < 3; ++y)
          o[3 * x + y] = hinv[3 * x] * r[y] + hinv[3 * x + 1] * r[3 + y] + hinv[3 * x + 2] * r[6 + y];
      for (int e = 0; e < 9; ++e) w.res[t * 9 + e] = o[e];
    }
    __syncthreads();
    if (threadIdx.x < 9) hfr[threadIdx.x] = w.res[(T - 1) * 9 + threadIdx.x];
    __syncthreads();
    const double* last = w.pts + (long long)(T - 1) * N * 2;
    double* dst = w.tformed + (long long)fr * N * 2;
    for (int n = threadIdx.x; n < N; n += kSolveThreads) {
      const Tf p = transform(hfr, last[2 * n], last[2 * n + 1], w.canon[2 * n], w.canon[2 * n + 1]);
      dst[2 * n] = p.x;
      dst[2 * n + 1] = p.y;
    }
    if (threadIdx.x < 9) s.h[threadIdx.x] = threadIdx.x % 4 == 0 ? 1.0 : 0.0;
    __syncthreads();
  }
  if (threadIdx.x < 9) {
    w.res[fr * 9 + threadIdx.x] = s.h[threadIdx.x];
    w.hcur[threadIdx.x] = s.h[threadIdx.x];
  }
}

// compute_canonical_points for 32 points per CTA, 16 warps over contiguous frame slices.  With
// apply_fr >= 0 it first transforms frame apply_fr with hcur (tformed, err; and, in the sweep, the
// frame's occlusion becomes its validity).  per_frame_err selects the [T][N] err form (the
// reference frame's branch) over the broadcast err of frame apply_fr.
__global__ void __launch_bounds__(kCanonWarps * 32) canonical_kernel(
    Ws w, int T, int N, int apply_fr, int sweep, int per_frame_err, int err_fr, int write_bad,
    unsigned call, double thresh, double required) {
  __shared__ double sx_[kCanonWarps][32], sy_[kCanonWarps][32];
  __shared__ int keep_[kCanonWarps][32], inl_[kCanonWarps][32], vis_[kCanonWarps][32];
  __shared__ int pick_warp[32], pick_id[32], pick_frame[32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int n = blockIdx.x * 32 + lane;
  const bool live = n < N;
  if (warp == 0 && live) {
    pick_frame[lane] = 0;
    if (apply_fr >= 0) {
      const long long idx = (long long)apply_fr * N + n;
      const Tf p = transform(w.hcur, w.pts[2 * idx], w.pts[2 * idx + 1], w.canon[2 * n], w.canon[2 * n + 1]);
      w.tformed[2 * idx] = p.x;
      w.tformed[2 * idx + 1] = p.y;
      w.err[idx] = p.err;
      if (sweep) w.inval[idx] = w.occ[idx];
    }
  }
  __syncthreads();
  const int per = (T + kCanonWarps - 1) / kCanonWarps;
  const int t0 = min(T, warp * per), t1 = min(T, t0 + per);
  const double outer = thresh * 2.0;
  double sx = 0.0, sy = 0.0;
  int keep = 0, inl = 0, vis = 0;
  if (live) {
    const double e_now = per_frame_err ? 0.0 : w.err[(long long)err_fr * N + n];
    for (int t = t0; t < t1; ++t) {
      const long long idx = (long long)t * N + n;
      const bool inv = w.inval[idx];
      const double e = per_frame_err ? w.err[idx] : e_now;
      const bool k = !(inv || e > outer);
      const double kd = k ? 1.0 : 0.0;
      sx += w.tformed[2 * idx] * kd;
      sy += w.tformed[2 * idx + 1] * kd;
      keep += k;
      inl += !inv && e < thresh;
      vis += !inv;
    }
  }
  sx_[warp][lane] = sx;
  sy_[warp][lane] = sy;
  keep_[warp][lane] = keep;
  inl_[warp][lane] = inl;
  vis_[warp][lane] = vis;
  __syncthreads();
  double px = 0.0, py = 0.0;
  bool bad = false;
  if (warp == 0 && live) {
    int nk = 0, ni = 0, nv = 0;
    for (int x = 0; x < kCanonWarps; ++x) {
      px += sx_[x][lane];
      py += sy_[x][lane];
      nk += keep_[x][lane];
      ni += inl_[x][lane];
      nv += vis_[x][lane];
    }
    const double frac = (double)ni / fmax(1.0, (double)nv);
    bad = frac < required;
    const double div = fmax(1.0, (double)nk);
    px /= div;
    py /= div;
    // the frame whose 1-based visible count is floor(u * count); frame 0 when that is 0
    const uint64_t bits = mix64(mix64(1) ^ (((uint64_t)call << 32) | (uint64_t)n)) >> 11;
    const double u = (double)bits * 0x1p-53;
    const int target = (int)floor(__dmul_rn(u, (double)nv));
    pick_warp[lane] = -1;
    if (target >= 1) {
      int before = 0;
      for (int x = 0; x < kCanonWarps; ++x) {
        if (target <= before + vis_[x][lane]) {
          pick_warp[lane] = x;
          pick_id[lane] = target - before;
          break;
        }
        before += vis_[x][lane];
      }
    }
  }
  __syncthreads();
  if (live && pick_warp[lane] == warp) {
    int seen = 0;
    for (int t = t0; t < t1; ++t) {
      seen += !w.inval[(long long)t * N + n];
      if (seen == pick_id[lane]) {
        pick_frame[lane] = t;
        break;
      }
    }
  }
  __syncthreads();
  if (warp == 0 && live) {
    const long long idx = (long long)pick_frame[lane] * N + n;
    const double b = bad ? 1.0 : 0.0, nb = bad ? 0.0 : 1.0;
    w.canon[2 * n] = __dadd_rn(__dmul_rn(b, w.tformed[2 * idx]), __dmul_rn(nb, px));
    w.canon[2 * n + 1] = __dadd_rn(__dmul_rn(b, w.tformed[2 * idx + 1]), __dmul_rn(nb, py));
    if (write_bad) w.cbad[n] = bad;
  }
}

// res @ diag(1 / width, 1 / height, 1), err transposed to [N][T], the canonical points.
__global__ void output_kernel(tapir_homography_args a, Ws w) {
  const int T = a.T, N = a.N;
  const double dg[3] = {1.0 / a.width, 1.0 / a.height, 1.0};
  const long long stride = (long long)gridDim.x * blockDim.x;
  const long long start = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  for (long long idx = start; idx < 9ll * T; idx += stride) {
    const double* r = w.res + idx / 9 * 9;
    const int row = (int)(idx % 9) / 3, col = (int)(idx % 3);
    double v = 0.0;
    for (int k = 0; k < 3; ++k) v = __dadd_rn(v, __dmul_rn(r[3 * row + k], k == col ? dg[col] : 0.0));
    a.homogs[idx] = v;
  }
  for (long long idx = start; idx < (long long)T * N; idx += stride) {
    const long long n = idx / T, t = idx % T;
    a.err[idx] = w.err[t * N + n];
  }
  for (long long idx = start; idx < 2ll * N; idx += stride) a.canonical[idx] = w.canon[idx];
}

}  // namespace

size_t homographies_workspace_bytes(int T, int N) {
  if (T < 1 || N < 1) return 0;
  Arena a(nullptr, 0);
  carve(a, T, N);
  return a.off;
}

void ransac_stop_thresholds(int N, double frac, double* out) {
  for (int it = 0; it < N; ++it) {
    const double a = 1.0 - (double)(it + 1) / (double)N;
    const double b = frac * pow(0.99, (double)it);
    out[it] = (b < a ? b : a) * (double)N;
  }
}

int homographies_wrt_frame(const tapir_homography_args* a, cudaStream_t s) {
  const int T = a->T, N = a->N, ref = a->reference_frame;
  Arena arena(a->workspace, a->workspace_bytes);
  const Ws w = carve(arena, T, N);
  const double t2 = a->thresh * a->thresh;
  const int canon_grid = (N + 31) / 32;
  const int score_grid = std::min(scan_blocks(N), kScoreCtas);
  const long long tn = (long long)T * N;
  const int init_grid = (int)std::min<long long>(std::max<long long>(ceil_div_ll(tn, 256), 1), 4096);
  unsigned call = 0;
  auto canonical = [&](int apply_fr, int sweep, int per_frame_err, int write_bad) {
    canonical_kernel<<<canon_grid, kCanonWarps * 32, 0, s>>>(
        w, T, N, apply_fr, sweep, per_frame_err, apply_fr, write_bad, ++call, a->thresh,
        a->outlier_point_threshold);
    count_launch();
  };
  init_kernel<<<init_grid, 256, 0, s>>>(*a, w);
  count_launch();
  TAPIR_LAUNCH_CHECK("homography init_kernel");
  // sweep order: the frames after the reference ascending, then those before it descending
  auto frame_at = [&](int x) { return x < T - 1 - ref ? ref + 1 + x : ref - 1 - (x - (T - 1 - ref)); };
  for (int x = 0; x < T - 1; ++x) {
    const int i = frame_at(x);
    prep_kernel<<<1, kPrepThreads, 0, s>>>(w, N, i);
    score_kernel<<<score_grid, kHypWarps * 32, 0, s>>>(w, a->stop_thresholds, N, i, t2);
    estimate_kernel<<<1, kSolveThreads, 0, s>>>(*a, w, i, t2);
    count_launch(3);
    canonical(i, 1, 0, 1);
    TAPIR_LAUNCH_CHECK("homography sweep kernels");
  }
  for (int j = 0; j < a->num_refinement_passes; ++j) {
    for (int x = -1; x < T - 1; ++x) {
      const int fr = x < 0 ? ref : frame_at(x);
      const int branch = fr == ref && j != a->num_refinement_passes - 1;
      refine_kernel<<<1, kSolveThreads, 0, s>>>(*a, w, fr, branch, t2);
      count_launch();
      if (branch) {
        // canonical points from every frame's own err; canonical_invalid is not updated
        canonical_kernel<<<canon_grid, kCanonWarps * 32, 0, s>>>(
            w, T, N, -1, 0, 1, 0, 0, ++call, a->thresh, a->outlier_point_threshold);
        count_launch();
      }
      canonical(fr, 0, 0, 1);
      TAPIR_LAUNCH_CHECK("homography refinement kernels");
    }
  }
  output_kernel<<<init_grid, 256, 0, s>>>(*a, w);
  count_launch();
  TAPIR_LAUNCH_CHECK("homography output_kernel");
  return kOk;
}

}  // namespace tapir
