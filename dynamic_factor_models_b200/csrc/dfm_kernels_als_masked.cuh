// dfm_kernels_als_masked.cuh -- fused ALS kernel for panels WITH missing data (no constraints):
// the reference's least-squares "EM" loop (estimate_factor!, dfm_functions.ipynb:352-370) for one panel per CTA, all
// sweeps in ONE launch -- no host synchronisation inside the sweep loop (the general kernels k_als_lambda /
// k_als_factor / k_als_check need a launch triple per sweep and a host read-back of the done flags).
//   Lambda-step (:355-362)  series i (>= nt_min observations, :357):  A_i = sum_{t obs} f_t f_t' = F'F - sum_{t miss} f_t f_t',
//                           b_i = sum_{t obs} x_it f_t,  lam_i = A_i^-1 b_i             (thread per series)
//   F-step      (:364-365)  period t:  A_t = Lam'Lam - sum_{i miss} lam_i lam_i',  b_t = sum_{i obs} x_it lam_i,
//                           f_t = A_t^-1 b_t                                            (thread per period)
//   SSR         (:366)      sum_{obs} (x - lam'f)^2 = sum_t (q_t - f_t'b_t),  q_t = sum_{i obs} x_it^2   (A_t f_t = b_t)
//   stop        (:367-368)  |dSSR| < tol T N
// With ~6 % missing cells the masked Gram matrices cost one rank-one DOWNDATE per missing cell instead of one update
// per observed cell.  The panel itself (T x N doubles, C1: 247 KB) is re-read by every step: a bootstrap batch
// keeps two panels per SM in flight (H100: 264 panels = 65 MB, somewhat more than the 50 MB L2).
// The r x r systems are solved in registers (packed Cholesky, fully unrolled for the template R).
#pragma once
#include "dfm_kernels_fused.cuh"

namespace dfm {

struct AlsMaskedArgs {
  const double* Xs;     // [B][N][T] standardised, NaN = missing
  double* F;            // [B][T*r] column-major: in = starting factors, out = final factors
  double* Lam;          // [B][N*r] column-major out (NaN rows: series with < nt_min observations)
  AlsState* st;         // tss / nobs already set; ssr, ssr_old, iters, done, status written here
  int B, T, N, nt_min;
  double tol;
  long long max_iter;
};

// packed lower Cholesky solve A x = b in registers (A: NP = R(R+1)/2 entries, row-major lower), fully unrolled.
template <int R>
__device__ __forceinline__ int reg_chol_solve(double (&A)[R * (R + 1) / 2], double (&b)[R]) {
  int bad = 0;
#pragma unroll
  for (int j = 0; j < R; ++j) {
    double d = A[j * (j + 1) / 2 + j];
#pragma unroll
    for (int c = 0; c < j; ++c) d -= A[j * (j + 1) / 2 + c] * A[j * (j + 1) / 2 + c];
    if (!(d > 0.0)) { bad = 1; d = 1.0; }
    d = sqrt(d);
    A[j * (j + 1) / 2 + j] = d;
    const double inv = 1.0 / d;
#pragma unroll
    for (int i = j + 1; i < R; ++i) {
      double s = A[i * (i + 1) / 2 + j];
#pragma unroll
      for (int c = 0; c < j; ++c) s -= A[i * (i + 1) / 2 + c] * A[j * (j + 1) / 2 + c];
      A[i * (i + 1) / 2 + j] = s * inv;
    }
  }
#pragma unroll
  for (int i = 0; i < R; ++i) {
    double s = b[i];
#pragma unroll
    for (int c = 0; c < i; ++c) s -= A[i * (i + 1) / 2 + c] * b[c];
    b[i] = s / A[i * (i + 1) / 2 + i];
  }
#pragma unroll
  for (int i = R - 1; i >= 0; --i) {
    double s = b[i];
#pragma unroll
    for (int c = i + 1; c < R; ++c) s -= A[c * (c + 1) / 2 + i] * b[c];
    b[i] = s / A[i * (i + 1) / 2 + i];
  }
  return bad;
}

#ifdef DFM_EMU
#define DFM_ALSM_BOUNDS
#else
#define DFM_ALSM_BOUNDS __launch_bounds__(256, 2)
#endif
template <int R>
__global__ void DFM_ALSM_BOUNDS k_als_masked(AlsMaskedArgs a) {
  DFM_SMEM(sm);
  constexpr int RR = R * R, NP = R * (R + 1) / 2;
  const int T = a.T, N = a.N;
  const int Tp = T | 1, Np = N | 1;            // odd leading dimensions: the R component rows start in different banks
  double* Fs = sm;                             // [R][Tp] component-major
  double* Ls = Fs + (size_t)R * Tp;            // [R][Np]
  double* G = Ls + (size_t)R * Np;             // [RR] F'F resp. Lam'Lam (full, row-major)
  double* part = G + RR;                       // [4][RR] partial Gram sums
  double* red = part + 4 * RR;                 // 40
  int* ctl = (int*)(red + 40);                 // [0] = status raised by a thread
  for (int b = DFM_BX; b < a.B; b += DFM_GX) {
    const double* X = a.Xs + (size_t)b * T * N;
    for (int e = DFM_TID; e < T * R; e += DFM_NT) { const int t = e % T, c = e / T; Fs[c * Tp + t] = a.F[(size_t)b * T * R + e]; }
    if (DFM_TID == 0) ctl[0] = 0;
    DFM_SYNC();
    double ssr = 0.0, ssr_old = 0.0;
    long long it = 0;
    int status = 0;
    while (it < a.max_iter) {
      // ---------------- Gram matrix of the factors (4 time slices per entry, fixed order)
      for (int e = DFM_TID; e < 4 * RR; e += DFM_NT) {
        const int sl = e / RR, ee = e % RR, i = ee / R, j = ee % R;
        const int t0 = (int)((long long)T * sl / 4), t1 = (int)((long long)T * (sl + 1) / 4);
        double s = 0.0;
        if (j <= i) for (int t = t0; t < t1; ++t) s += Fs[i * Tp + t] * Fs[j * Tp + t];
        part[e] = s;
      }
      DFM_SYNC();
      for (int e = DFM_TID; e < RR; e += DFM_NT) { const int i = e / R, j = e % R; const int lo = (j <= i) ? e : j * R + i; G[e] = part[lo] + part[RR + lo] + part[2 * RR + lo] + part[3 * RR + lo]; }
      DFM_SYNC();
      // ---------------- Lambda-step: thread per series
      for (int i = DFM_TID; i < N; i += DFM_NT) {
        const double* x = X + (size_t)i * T;
        double A[NP], c[R];
#pragma unroll
        for (int e = 0; e < NP; ++e) A[e] = 0.0;
#pragma unroll
        for (int q = 0; q < R; ++q) c[q] = 0.0;
        int cnt = 0;
        // the panel comes from L2 (long latency per load): eight loads in flight per thread, then the arithmetic -- the
        // branchy one-load-per-iteration loop waited a full round trip for every cell
        for (int t0 = 0; t0 < T; t0 += 8) {
          double vv[8];
#pragma unroll
          for (int u = 0; u < 8; ++u) vv[u] = (t0 + u < T) ? x[t0 + u] : 0.0;
#pragma unroll
          for (int u = 0; u < 8; ++u) {
            const int t = t0 + u;
            if (t < T) {
              const double v = vv[u];
              if (!is_nan(v)) {
                ++cnt;
#pragma unroll
                for (int q = 0; q < R; ++q) c[q] += v * Fs[q * Tp + t];
              } else {
                double f[R];
#pragma unroll
                for (int q = 0; q < R; ++q) f[q] = Fs[q * Tp + t];
#pragma unroll
                for (int q = 0; q < R; ++q)
#pragma unroll
                  for (int p = 0; p <= q; ++p) A[q * (q + 1) / 2 + p] += f[q] * f[p];
              }
            }
          }
        }
        bool ok = cnt >= a.nt_min;
        if (ok) {
#pragma unroll
          for (int q = 0; q < R; ++q)
#pragma unroll
            for (int p = 0; p <= q; ++p) A[q * (q + 1) / 2 + p] = G[q * R + p] - A[q * (q + 1) / 2 + p];
          if (reg_chol_solve<R>(A, c)) { ctl[0] = 3; ok = false; }
        }
#pragma unroll
        for (int q = 0; q < R; ++q) Ls[q * Np + i] = ok ? c[q] : DFM_NAN;
      }
      DFM_SYNC();
      // ---------------- Gram matrix of the loadings (series in the model only)
      for (int e = DFM_TID; e < 4 * RR; e += DFM_NT) {
        const int sl = e / RR, ee = e % RR, i = ee / R, j = ee % R;
        const int n0 = (int)((long long)N * sl / 4), n1 = (int)((long long)N * (sl + 1) / 4);
        double s = 0.0;
        if (j <= i) for (int n = n0; n < n1; ++n) { const double li = Ls[i * Np + n]; if (!is_nan(Ls[n])) s += li * Ls[j * Np + n]; }
        part[e] = s;
      }
      DFM_SYNC();
      for (int e = DFM_TID; e < RR; e += DFM_NT) { const int i = e / R, j = e % R; const int lo = (j <= i) ? e : j * R + i; G[e] = part[lo] + part[RR + lo] + part[2 * RR + lo] + part[3 * RR + lo]; }
      DFM_SYNC();
      // ---------------- F-step: thread per period (reads of X are coalesced across the threads)
      double ssr_p = 0.0;
      for (int t = DFM_TID; t < T; t += DFM_NT) {
        double A[NP], c[R], q2 = 0.0;
#pragma unroll
        for (int e = 0; e < NP; ++e) A[e] = 0.0;
#pragma unroll
        for (int q = 0; q < R; ++q) c[q] = 0.0;
        int nobs = 0;
        for (int i0 = 0; i0 < N; i0 += 8) {                         // (eight cells of the period in flight, see above)
          double vv[8];
#pragma unroll
          for (int u = 0; u < 8; ++u) vv[u] = (i0 + u < N) ? X[(size_t)(i0 + u) * T + t] : 0.0;
#pragma unroll
          for (int u = 0; u < 8; ++u) {
            const int i = i0 + u;
            if (i < N) {
              const double l0 = Ls[i];
              if (!is_nan(l0)) {
                const double v = vv[u];
                if (!is_nan(v)) {
                  ++nobs; q2 += v * v;
#pragma unroll
                  for (int q = 0; q < R; ++q) c[q] += v * Ls[q * Np + i];
                } else {
                  double l[R];
#pragma unroll
                  for (int q = 0; q < R; ++q) l[q] = Ls[q * Np + i];
#pragma unroll
                  for (int q = 0; q < R; ++q)
#pragma unroll
                    for (int p = 0; p <= q; ++p) A[q * (q + 1) / 2 + p] += l[q] * l[p];
                }
              }
            }
          }
        }
#pragma unroll
        for (int q = 0; q < R; ++q)
#pragma unroll
          for (int p = 0; p <= q; ++p) A[q * (q + 1) / 2 + p] = G[q * R + p] - A[q * (q + 1) / 2 + p];
        double bt[R];
#pragma unroll
        for (int q = 0; q < R; ++q) bt[q] = c[q];
        int bad = (nobs < R) ? 2 : (reg_chol_solve<R>(A, c) ? 3 : 0);
        if (bad) { ctl[0] = bad; 
#pragma unroll
          for (int q = 0; q < R; ++q) c[q] = DFM_NAN; }
        else { double fb = 0.0;
#pragma unroll
          for (int q = 0; q < R; ++q) fb += c[q] * bt[q];
          ssr_p += q2 - fb; }
#pragma unroll
        for (int q = 0; q < R; ++q) Fs[q * Tp + t] = c[q];
      }
      ssr_p = block_sum(ssr_p, red);
      ssr_old = ssr; ssr = ssr_p;
      ++it;
      if (ctl[0]) { status = ctl[0]; break; }
      if (!(fabs(ssr_old - ssr) >= a.tol * (double)T * (double)N)) break;            // :367-368
      if (it >= a.max_iter) { status = 4; break; }
    }
    for (int e = DFM_TID; e < T * R; e += DFM_NT) { const int t = e % T, c = e / T; a.F[(size_t)b * T * R + e] = Fs[c * Tp + t]; }
    for (int e = DFM_TID; e < N * R; e += DFM_NT) { const int i = e % N, c = e / N; a.Lam[(size_t)b * N * R + e] = Ls[c * Np + i]; }
    if (DFM_TID == 0) { a.st[b].ssr_old = ssr_old; a.st[b].ssr = ssr; a.st[b].iters = (int)it; a.st[b].done = 1; a.st[b].status = status; }
    DFM_SYNC();
  }
}

template <int R>
inline size_t als_masked_smem_doubles(int T, int N) {
  return (size_t)R * (T | 1) + (size_t)R * (N | 1) + 5 * (size_t)R * R + 40 + 8;
}

}  // namespace dfm
