// dfm_common.cuh -- launch/sync abstraction + block-cooperative small dense FP64 helpers.
//
// Product build: nvcc -gencode arch=compute_90a,code=sm_90a (real CUDA, H100).
// DFM_EMU build (tests/emu only, never shipped or loaded by the package): the SAME kernel
// source compiled by g++ with one "thread" per block, so index/algebra logic can be checked in
// the GPU-less build container.  It is a test harness for the kernel source, not a fallback:
// libdfm_b200.so contains no host compute path.
#pragma once
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>

#ifdef DFM_EMU
// ------------------------------------------------------------------ host emulation layer
#include <cstdlib>
#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define __restrict__
struct dfm_emu_ctx { int bx, by, gx, gy; };
static thread_local dfm_emu_ctx g_emu;
static thread_local double g_emu_smem[1 << 19];   // 4 MB of "shared memory"
#define DFM_TID 0
#define DFM_NT 1
#define DFM_BX (g_emu.bx)
#define DFM_BY (g_emu.by)
#define DFM_GX (g_emu.gx)
#define DFM_SYNC() ((void)0)
#define DFM_SMEM(name) double* name = g_emu_smem
static inline double atomicAdd(double* p, double v) { double o = *p; *p += v; return o; }
static inline int atomicAdd(int* p, int v) { int o = *p; *p += v; return o; }
static inline int atomicMax(int* p, int v) { int o = *p; if (v > o) *p = v; return o; }
static inline int atomicMin(int* p, int v) { int o = *p; if (v < o) *p = v; return o; }
typedef void* cudaStream_t;
#define DFM_LAUNCH(kern, gx_, gy_, nt_, smem_, stream_, ...)                          \
  do {                                                                               \
    g_emu.gx = (gx_); g_emu.gy = (gy_);                                              \
    for (int by__ = 0; by__ < (gy_); ++by__)                                         \
      for (int bx__ = 0; bx__ < (gx_); ++bx__) { g_emu.bx = bx__; g_emu.by = by__; kern(__VA_ARGS__); } \
  } while (0)
#else
// ------------------------------------------------------------------ real CUDA
#include <cuda_runtime.h>
#define DFM_TID ((int)threadIdx.x)
#define DFM_NT ((int)blockDim.x)
#define DFM_BX ((int)blockIdx.x)
#define DFM_BY ((int)blockIdx.y)
#define DFM_GX ((int)gridDim.x)
#define DFM_SYNC() __syncthreads()
#define DFM_SMEM(name) extern __shared__ double name[]
#define DFM_LAUNCH(kern, gx_, gy_, nt_, smem_, stream_, ...) \
  kern<<<dim3((unsigned)(gx_), (unsigned)(gy_)), (unsigned)(nt_), (size_t)(smem_), (stream_)>>>(__VA_ARGS__)
#endif

#define DFM_NAN (nan(""))

// warp-level view of the block (the host emulation runs one logical thread per block)
#ifdef DFM_EMU
#define DFM_LANE 0
#define DFM_WSZ 1
#define DFM_WARP 0
#define DFM_NWARP 1
#define DFM_WSYNC() ((void)0)
#else
#define DFM_LANE ((int)(threadIdx.x & 31))
#define DFM_WSZ 32
#define DFM_WARP ((int)(threadIdx.x >> 5))
#define DFM_NWARP ((int)(blockDim.x >> 5))
#define DFM_WSYNC() __syncwarp()
#endif


namespace dfm {

__device__ __forceinline__ bool is_nan(double x) { return x != x; }

// Sum over the block.  `red` = >= 33 doubles of shared scratch.  All threads get the result.
__device__ __forceinline__ double block_sum(double v, double* red) {
#ifdef DFM_EMU
  (void)red;
  return v;
#else
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  if (lane == 0) red[w] = v;
  __syncthreads();
  if (w == 0) {
    double s = (lane < nw) ? red[lane] : 0.0;
    for (int o = 16; o > 0; o >>= 1) s += __shfl_down_sync(0xffffffffu, s, o);
    if (lane == 0) red[32] = s;
  }
  __syncthreads();
  double out = red[32];
  __syncthreads();
  return out;
#endif
}

// packed lower-triangular index, a >= c
__device__ __forceinline__ int pidx(int a, int c) { return a * (a + 1) / 2 + c; }

// ---- thread-private solve: packed lower SPD matrix A (element (a,c) at A[pidx(a,c)*stride]),
// rhs b (b[a*stride]); overwrites A with its Cholesky factor and b with the solution.
// returns 0 ok, 1 not PD.
__device__ inline int chol_solve_packed(double* A, double* b, int n, int stride) {
  for (int j = 0; j < n; ++j) {
    double d = A[pidx(j, j) * stride];
    for (int c = 0; c < j; ++c) { double l = A[pidx(j, c) * stride]; d -= l * l; }
    if (!(d > 0.0)) return 1;
    d = sqrt(d);
    A[pidx(j, j) * stride] = d;
    double inv = 1.0 / d;
    for (int i = j + 1; i < n; ++i) {
      double s = A[pidx(i, j) * stride];
      for (int c = 0; c < j; ++c) s -= A[pidx(i, c) * stride] * A[pidx(j, c) * stride];
      A[pidx(i, j) * stride] = s * inv;
    }
  }
  for (int i = 0; i < n; ++i) {          // L y = b
    double s = b[i * stride];
    for (int c = 0; c < i; ++c) s -= A[pidx(i, c) * stride] * b[c * stride];
    b[i * stride] = s / A[pidx(i, i) * stride];
  }
  for (int i = n - 1; i >= 0; --i) {     // L' x = y
    double s = b[i * stride];
    for (int c = i + 1; c < n; ++c) s -= A[pidx(c, i) * stride] * b[c * stride];
    b[i * stride] = s / A[pidx(i, i) * stride];
  }
  return 0;
}

// solve with an already factored packed lower L (as left by chol_solve_packed)
__device__ inline void chol_resolve_packed(const double* L, double* b, int n, int stride) {
  for (int i = 0; i < n; ++i) {
    double s = b[i * stride];
    for (int c = 0; c < i; ++c) s -= L[pidx(i, c) * stride] * b[c * stride];
    b[i * stride] = s / L[pidx(i, i) * stride];
  }
  for (int i = n - 1; i >= 0; --i) {
    double s = b[i * stride];
    for (int c = i + 1; c < n; ++c) s -= L[pidx(c, i) * stride] * b[c * stride];
    b[i * stride] = s / L[pidx(i, i) * stride];
  }
}

// ================= block-cooperative dense ops on column-major matrices (shared or global) =====
// Every routine ends with DFM_SYNC(); outputs must not alias inputs unless stated.

// C(m x n) = beta*C + alpha * opA(A) * opB(B);  opA(A) is m x kk, opB(B) is kk x n.
__device__ inline void bm_gemm(double* C, int ldc, const double* A, int lda, bool ta, const double* B, int ldb,
                               bool tb, int m, int n, int kk, double alpha, double beta) {
  for (int e = DFM_TID; e < m * n; e += DFM_NT) {
    int i = e % m, j = e / m;
    double s = 0.0;
    for (int l = 0; l < kk; ++l) {
      double a = ta ? A[l + lda * i] : A[i + lda * l];
      double b = tb ? B[j + ldb * l] : B[l + ldb * j];
      s += a * b;
    }
    double c0 = (beta == 0.0) ? 0.0 : beta * C[i + ldc * j];
    C[i + ldc * j] = c0 + alpha * s;
  }
  DFM_SYNC();
}

__device__ inline void bm_copy(double* D, int ldd, const double* S, int lds, int m, int n) {
  for (int e = DFM_TID; e < m * n; e += DFM_NT) { int i = e % m, j = e / m; D[i + ldd * j] = S[i + lds * j]; }
  DFM_SYNC();
}

// A <- (A + A')/2  (n x n)
__device__ inline void bm_symmetrize(double* A, int ld, int n) {
  for (int e = DFM_TID; e < n * n; e += DFM_NT) {
    int i = e % n, j = e / n;
    if (i > j) { double v = 0.5 * (A[i + ld * j] + A[j + ld * i]); A[i + ld * j] = v; A[j + ld * i] = v; }
  }
  DFM_SYNC();
}

// In-place lower Cholesky of the n x n SPD matrix A (upper triangle is ZEROED so A can be used
// as a full matrix afterwards).  *info (shared int) is set to 1 on a non-positive pivot.
// Right-looking with ONE barrier per column: the columns stay unscaled during the elimination (the trailing
// update divides by the pivot d_j instead), and are scaled by 1/sqrt(d_j) in one pass at the end.
__device__ inline void bm_chol(double* A, int ld, int n, int* info) {
  for (int j = 0; j < n; ++j) {
    double d = A[j + ld * j];                        // final after the updates of columns < j
    if (!(d > 0.0)) { if (DFM_TID == 0) *info = 1; d = 1.0; }
    const double dinv = 1.0 / d;
    const int m = n - j - 1;                         // trailing update of the lower triangle, columns j+1..n-1
    for (int e = DFM_TID; e < m * m; e += DFM_NT) {
      int i = j + 1 + e % m, c = j + 1 + e / m;
      if (i >= c) A[i + ld * c] -= A[i + ld * j] * A[c + ld * j] * dinv;
    }
    DFM_SYNC();
  }
  for (int e = DFM_TID; e < n * n; e += DFM_NT) {
    int i = e % n, j = e / n;
    if (i < j) { A[i + ld * j] = 0.0; continue; }
    double d = A[j + ld * j];
    if (!(d > 0.0)) d = 1.0;
    if (i > j) A[i + ld * j] *= 1.0 / sqrt(d);
  }
  DFM_SYNC();
  for (int j = DFM_TID; j < n; j += DFM_NT) { double d = A[j + ld * j]; if (!(d > 0.0)) d = 1.0; A[j + ld * j] = sqrt(d); }
  DFM_SYNC();
}

// B (n x m) <- L^-1 B   (L lower, n x n).  Right-looking, all threads on the rank-one update of the rows below the
// pivot row, ONE barrier per row: rows stay unscaled during the elimination (x_i = B_i / L_ii is formed on the fly)
// and are divided by the diagonal in one pass at the end.
__device__ inline void bm_trsm_lower(const double* L, int ldl, int n, double* B, int ldb, int m) {
  for (int i = 0; i + 1 < n; ++i) {
    const double inv = 1.0 / L[i + ldl * i];
    const int nr = n - i - 1;
    for (int e = DFM_TID; e < nr * m; e += DFM_NT) {
      int i2 = i + 1 + e % nr, c = e / nr;
      B[i2 + ldb * c] -= L[i2 + ldl * i] * (B[i + ldb * c] * inv);
    }
    DFM_SYNC();
  }
  for (int e = DFM_TID; e < n * m; e += DFM_NT) { int i = e % n, c = e / n; B[i + ldb * c] /= L[i + ldl * i]; }
  DFM_SYNC();
}

// B (n x m) <- L^-T B
__device__ inline void bm_trsm_lowerT(const double* L, int ldl, int n, double* B, int ldb, int m) {
  for (int i = n - 1; i > 0; --i) {
    const double inv = 1.0 / L[i + ldl * i];
    for (int e = DFM_TID; e < i * m; e += DFM_NT) {
      int i2 = e % i, c = e / i;
      B[i2 + ldb * c] -= L[i + ldl * i2] * (B[i + ldb * c] * inv);
    }
    DFM_SYNC();
  }
  for (int e = DFM_TID; e < n * m; e += DFM_NT) { int i = e % n, c = e / n; B[i + ldb * c] /= L[i + ldl * i]; }
  DFM_SYNC();
}

// ================= fast reciprocals, block-cooperative Cholesky, transposed solves, tensor-core tile products =========
// Reciprocal and reciprocal square root from the hardware seed (MUFU, ~2^-23) + two Newton steps: ~1 ulp, a fraction of
// the latency of the correctly rounded division / sqrt sequences, which sit on the serial path of every Cholesky column.
__device__ __forceinline__ double fast_rcp(double d) {
#ifdef DFM_EMU
  return 1.0 / d;
#else
  double y;
  asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(d));
  double e = fma(-d, y, 1.0); y = fma(y, e, y);        // 2^-23 -> 2^-46
  e = fma(-d, y, 1.0); y = fma(y, e, y);               // -> below 2^-53 (~1 ulp after rounding)
  return y;
#endif
}
__device__ __forceinline__ double fast_rsqrt(double d) {
#ifdef DFM_EMU
  return 1.0 / sqrt(d);
#else
  double y;
  asm("rsqrt.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(d));
  const double hd = 0.5 * d;
  double e = fma(-hd * y, y, 0.5); y = fma(y, e, y);
  e = fma(-hd * y, y, 0.5); y = fma(y, e, y);
  return y;
#endif
}

// Lower Cholesky of the n x n SPD matrix A (shared, column-major), block-cooperative, ONE barrier per column: columns stay
// unscaled during the elimination (the trailing update multiplies by 1/d_j), warps take the trailing columns, lanes the
// rows (conflict-free, no index arithmetic); one final pass scales column j by d_j^-1/2 and zeroes the upper triangle.
// dinv (n doubles, shared) receives 1 / L_jj for the triangular solves.  *info = 1 on a non-positive pivot.
__device__ inline void bc_chol(double* A, int ld, int n, double* dinv, int* info) {
  for (int j = 0; j < n; ++j) {
    double d = A[j + ld * j];                          // final after the updates of columns < j
    if (!(d > 0.0)) { if (DFM_TID == 0) *info = 1; d = 1.0; }
    const double di = fast_rcp(d);
    if (DFM_TID == 0) dinv[j] = d;                     // (pivot; turned into 1 / L_jj below)
    for (int c = j + 1 + DFM_WARP; c < n; c += DFM_NWARP) {
      const double lc = A[c + ld * j] * di;
      for (int i = c + DFM_LANE; i < n; i += DFM_WSZ) A[i + ld * c] -= A[i + ld * j] * lc;
    }
    DFM_SYNC();
  }
  for (int j = DFM_WARP; j < n; j += DFM_NWARP) {
    const double rs = fast_rsqrt(dinv[j]);
    for (int i = DFM_LANE; i < n; i += DFM_WSZ) {
      if (i < j) A[i + ld * j] = 0.0;
      else if (i == j) A[i + ld * j] = dinv[j] * rs;
      else A[i + ld * j] *= rs;
    }
  }
  DFM_SYNC();
  for (int j = DFM_TID; j < n; j += DFM_NT) dinv[j] = fast_rsqrt(dinv[j]);
  DFM_SYNC();
}

// Triangular solves on TRANSPOSED right-hand sides: XT is m x n (leading dimension ldx), ROW j of XT is the j-th right-hand
// side and is overwritten by its solution.  One thread per row, no barriers inside: consecutive threads touch consecutive
// addresses (conflict-free), the entries of L and 1 / L_aa (dinv) are warp-uniform broadcasts.  For n <= 32 the row lives
// in REGISTERS for the whole substitution (fully unrolled over a compile-time bound with uniform guards): re-reading the
// freshly stored components from shared memory put a store -> load round trip on every step of the serial chain.
#ifndef DFM_EMU
template <int NMAX, bool TRANS>
__device__ __noinline__ void bt_trsm_reg(const double* L, int ldl, int n, const double* dinv, double* XT, int ldx, int m) {
  for (int j = DFM_TID; j < m; j += DFM_NT) {
    double x[NMAX];
#pragma unroll
    for (int a = 0; a < NMAX; ++a) x[a] = (a < n) ? XT[j + ldx * a] : 0.0;
    if (!TRANS) {
#pragma unroll
      for (int a = 0; a < NMAX; ++a) {
        if (a < n) {
          double s0 = x[a], s1 = 0.0, s2 = 0.0, s3 = 0.0;
#pragma unroll
          for (int c = 0; c < a; ++c) {
            const double t = L[a + ldl * c] * x[c];
            if ((c & 3) == 0) s0 -= t; else if ((c & 3) == 1) s1 -= t; else if ((c & 3) == 2) s2 -= t; else s3 -= t;
          }
          x[a] = ((s0 + s1) + (s2 + s3)) * dinv[a];
        }
      }
    } else {
#pragma unroll
      for (int a = NMAX - 1; a >= 0; --a) {
        if (a < n) {
          double s0 = x[a], s1 = 0.0, s2 = 0.0, s3 = 0.0;
#pragma unroll
          for (int c = a + 1; c < NMAX; ++c) {
            const double t = (c < n) ? L[c + ldl * a] * x[c] : 0.0;
            if ((c & 3) == 0) s0 -= t; else if ((c & 3) == 1) s1 -= t; else if ((c & 3) == 2) s2 -= t; else s3 -= t;
          }
          x[a] = ((s0 + s1) + (s2 + s3)) * dinv[a];
        }
      }
    }
#pragma unroll
    for (int a = 0; a < NMAX; ++a) if (a < n) XT[j + ldx * a] = x[a];
  }
}
#endif
__device__ inline void bt_trsm_lower(const double* L, int ldl, int n, const double* dinv, double* XT, int ldx, int m) {      // L y = x
#ifndef DFM_EMU
  if (n <= 8) { bt_trsm_reg<8, false>(L, ldl, n, dinv, XT, ldx, m); DFM_SYNC(); return; }
  if (n <= 16) { bt_trsm_reg<16, false>(L, ldl, n, dinv, XT, ldx, m); DFM_SYNC(); return; }
  if (n <= 32) { bt_trsm_reg<32, false>(L, ldl, n, dinv, XT, ldx, m); DFM_SYNC(); return; }
#endif
  for (int j = DFM_TID; j < m; j += DFM_NT)
    for (int a = 0; a < n; ++a) {
      double s0 = XT[j + ldx * a], s1 = 0.0, s2 = 0.0, s3 = 0.0;
      int c = 0;
      for (; c + 3 < a; c += 4) {
        s0 -= L[a + ldl * c] * XT[j + ldx * c]; s1 -= L[a + ldl * (c + 1)] * XT[j + ldx * (c + 1)];
        s2 -= L[a + ldl * (c + 2)] * XT[j + ldx * (c + 2)]; s3 -= L[a + ldl * (c + 3)] * XT[j + ldx * (c + 3)];
      }
      for (; c < a; ++c) s0 -= L[a + ldl * c] * XT[j + ldx * c];
      XT[j + ldx * a] = ((s0 + s1) + (s2 + s3)) * dinv[a];
    }
  DFM_SYNC();
}
__device__ inline void bt_trsm_lowerT(const double* L, int ldl, int n, const double* dinv, double* XT, int ldx, int m) {     // L' y = x
  for (int j = DFM_TID; j < m; j += DFM_NT)
    for (int a = n - 1; a >= 0; --a) {
      double s0 = XT[j + ldx * a], s1 = 0.0, s2 = 0.0, s3 = 0.0;
      int c = a + 1;
      for (; c + 3 < n; c += 4) {
        s0 -= L[c + ldl * a] * XT[j + ldx * c]; s1 -= L[c + 1 + ldl * a] * XT[j + ldx * (c + 1)];
        s2 -= L[c + 2 + ldl * a] * XT[j + ldx * (c + 2)]; s3 -= L[c + 3 + ldl * a] * XT[j + ldx * (c + 3)];
      }
      for (; c < n; ++c) s0 -= L[c + ldl * a] * XT[j + ldx * c];
      XT[j + ldx * a] = ((s0 + s1) + (s2 + s3)) * dinv[a];
    }
  DFM_SYNC();
}

// Warp-tiled FP64 tensor-core product on shared-memory operands (mma.sync.m8n8k4.f64 -> DMMA.8x8x4):
//   D(m, n) = sum_l A(m, l) B(n, l),   A(m, l) = As[m * sam + l * sal],   B(n, l) = Bs[n * sbn + l * sbl],   m < Mr, n < Nn, l < K.
// The 8 x 8 output tiles are dealt to the warps round-robin; epi(m, n, value) is called once for every valid element.
// A dot-product loop on shared-memory operands needs two 8-byte operand reads per multiply-add and is bound by the
// shared-memory pipe (measured: the k x k products of the frozen-run phases); a DMMA needs two reads per 256 of them.
#ifndef DFM_EMU
#define EM_DMMA(d_, a_, b_) asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n" : "+d"((d_)[0]), "+d"((d_)[1]) : "d"(a_), "d"(b_))
#endif
template <class Epi>
__device__ __forceinline__ void wt_gemm(const double* As, int sam, int sal, const double* Bs, int sbn, int sbl, int Mr, int Nn, int K, Epi epi) {
#ifndef DFM_EMU
  const int lr = DFM_LANE >> 2, lc = DFM_LANE & 3;
  const int mt = (Mr + 7) >> 3, ntl = (Nn + 7) >> 3;
  for (int tile = DFM_WARP; tile < mt * ntl; tile += DFM_NWARP) {
    const int mb = tile % mt, nb = tile / mt;
    const int m = mb * 8 + lr, n = nb * 8 + lr;
    const bool mok = m < Mr, nok = n < Nn;
    const double* ap = As + (size_t)(mok ? m : 0) * sam + (size_t)lc * sal;
    const double* bp = Bs + (size_t)(nok ? n : 0) * sbn + (size_t)lc * sbl;
    double d0[2] = {0.0, 0.0}, d1[2] = {0.0, 0.0};
    int l0 = 0;
    for (; l0 + 8 <= K; l0 += 8) {
      const double a0 = mok ? ap[(size_t)l0 * sal] : 0.0, b0 = nok ? bp[(size_t)l0 * sbl] : 0.0;
      const double a1 = mok ? ap[(size_t)(l0 + 4) * sal] : 0.0, b1 = nok ? bp[(size_t)(l0 + 4) * sbl] : 0.0;
      EM_DMMA(d0, a0, b0); EM_DMMA(d1, a1, b1);
    }
    for (; l0 < K; l0 += 4) {
      const bool lok = l0 + lc < K;
      const double a0 = (mok && lok) ? ap[(size_t)l0 * sal] : 0.0, b0 = (nok && lok) ? bp[(size_t)l0 * sbl] : 0.0;
      EM_DMMA(d0, a0, b0);
    }
    const int mo = mb * 8 + lr, no = nb * 8 + 2 * lc;
    if (mo < Mr) { if (no < Nn) epi(mo, no, d0[0] + d1[0]); if (no + 1 < Nn) epi(mo, no + 1, d0[1] + d1[1]); }
  }
#else
  for (int n = 0; n < Nn; ++n)
    for (int m = 0; m < Mr; ++m) {
      double v = 0.0;
      for (int l = 0; l < K; ++l) v += As[(size_t)m * sam + (size_t)l * sal] * Bs[(size_t)n * sbn + (size_t)l * sbl];
      epi(m, n, v);
    }
#endif
}
// Same product accumulated into per-warp register tiles that persist over several calls (the reduction dimension arrives
// in pieces): tile index = warp + q * (number of warps), q < EM_TQ; acc[q] is the lane's pair of the tile's 8 x 8 block.
#define EM_TQ 6
__device__ __forceinline__ void wt_gemm_acc(const double* As, int sam, int sal, const double* Bs, int sbn, int sbl, int Mr, int Nn, int K,
                                            int tile0, double (*acc)[2]) {
#ifndef DFM_EMU
  const int lr = DFM_LANE >> 2, lc = DFM_LANE & 3;
  const int mt = (Mr + 7) >> 3, ntl = (Nn + 7) >> 3;
#pragma unroll
  for (int q = 0; q < EM_TQ; ++q) {
    const int tile = DFM_WARP + q * DFM_NWARP - tile0;
    if (tile >= 0 && tile < mt * ntl) {
      const int mb = tile % mt, nb = tile / mt;
      const int m = mb * 8 + lr, n = nb * 8 + lr;
      const bool mok = m < Mr, nok = n < Nn;
      const double* ap = As + (size_t)(mok ? m : 0) * sam + (size_t)lc * sal;
      const double* bp = Bs + (size_t)(nok ? n : 0) * sbn + (size_t)lc * sbl;
      for (int l0 = 0; l0 < K; l0 += 4) {
        const bool lok = l0 + lc < K;
        const double a0 = (mok && lok) ? ap[(size_t)l0 * sal] : 0.0, b0 = (nok && lok) ? bp[(size_t)l0 * sbl] : 0.0;
        EM_DMMA(acc[q], a0, b0);
      }
    }
  }
#else
  (void)As; (void)sam; (void)sal; (void)Bs; (void)sbn; (void)sbl; (void)Mr; (void)Nn; (void)K; (void)tile0; (void)acc;
#endif
}
// visit the elements of the register tiles: f(q-th tile's (m, n), value)
template <class F>
__device__ __forceinline__ void wt_acc_visit(int Mr, int Nn, int tile0, double (*acc)[2], F f) {
#ifndef DFM_EMU
  const int lr = DFM_LANE >> 2, lc = DFM_LANE & 3;
  const int mt = (Mr + 7) >> 3, ntl = (Nn + 7) >> 3;
#pragma unroll
  for (int q = 0; q < EM_TQ; ++q) {
    const int tile = DFM_WARP + q * DFM_NWARP - tile0;
    if (tile >= 0 && tile < mt * ntl) {
      const int mo = (tile % mt) * 8 + lr, no = (tile / mt) * 8 + 2 * lc;
      if (mo < Mr) { if (no < Nn) f(mo, no, acc[q][0]); if (no + 1 < Nn) f(mo, no + 1, acc[q][1]); }
    }
  }
#else
  (void)Mr; (void)Nn; (void)tile0; (void)acc; (void)f;
#endif
}
__host__ __device__ inline int em_lds(int k) { return k + ((12 - k % 8) % 8); }      // row stride == 4 (mod 8): conflict-free fragments

}  // namespace dfm
