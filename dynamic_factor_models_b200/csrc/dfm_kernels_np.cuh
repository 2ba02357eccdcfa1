// dfm_kernels_np.cuh -- kernels of the NON-PARAMETRIC path (rows a2..a11 of SURVEY.md section 8):
// standardise, PCA (Gram + Jacobi), ALS / least-squares-EM sweep, loadings + idiosyncratic AR,
// factor VAR + companion form, IRF.  All FP64, column-major, batched over blockIdx.y = panel.
// Reference lines cited as dfm_functions.ipynb:<raw JSON line>.
#pragma once
#include "dfm_common.cuh"

namespace dfm {

struct AlsState {          // one per panel, device resident
  double ssr, ssr_old, tss;
  long long nobs;
  int iters, done, status, pad;
};

// ---------------------------------------------------------------- K1 standardize_data :501-509
// grid (N, B); block per column.  Also per-column sum of squares / count for tss, nobs (:342-343).
__global__ void k_standardize(const double* __restrict__ X, int T, int N, double* __restrict__ Xs,
                              double* __restrict__ xmean, double* __restrict__ xstd,
                              double* __restrict__ col_ss, int* __restrict__ col_n) {
  DFM_SMEM(sm);
  int i = DFM_BX, b = DFM_BY;
  const double* x = X + ((size_t)b * N + i) * T;
  double* xs = Xs + ((size_t)b * N + i) * T;
  double s = 0.0, n = 0.0;
  for (int t = DFM_TID; t < T; t += DFM_NT) { double v = x[t]; if (!is_nan(v)) { s += v; n += 1.0; } }
  s = block_sum(s, sm); n = block_sum(n, sm);
  double mean = (n > 0) ? s / n : DFM_NAN;
  double v2 = 0.0;
  for (int t = DFM_TID; t < T; t += DFM_NT) { double v = x[t]; if (!is_nan(v)) { double d = v - mean; v2 += d * d; } }
  v2 = block_sum(v2, sm);
  double sd = (n > 0) ? sqrt(v2 / n) : DFM_NAN;      // population std  (:504-506)
  double ss = 0.0;
  for (int t = DFM_TID; t < T; t += DFM_NT) {
    double v = (x[t] - mean) / sd;
    xs[t] = v;
    if (!is_nan(v)) ss += v * v;
  }
  ss = block_sum(ss, sm);
  if (DFM_TID == 0) {
    if (xmean) xmean[(size_t)b * N + i] = mean;
    if (xstd) xstd[(size_t)b * N + i] = sd;
    if (col_ss) col_ss[(size_t)b * N + i] = ss;
    if (col_n) col_n[(size_t)b * N + i] = (int)n;
  }
}

// tss / nobs totals + state reset.  grid (B), 1 block.
__global__ void k_als_init_state(AlsState* st, const double* col_ss, const int* col_n, int N) {
  DFM_SMEM(sm);
  int b = DFM_BX;
  double ss = 0.0, n = 0.0;
  for (int i = DFM_TID; i < N; i += DFM_NT) { ss += col_ss[(size_t)b * N + i]; n += col_n[(size_t)b * N + i]; }
  ss = block_sum(ss, sm); n = block_sum(n, sm);
  if (DFM_TID == 0) {
    st[b].tss = ss; st[b].nobs = (long long)n; st[b].ssr = 0.0; st[b].ssr_old = 0.0;
    st[b].iters = 0; st[b].done = 0; st[b].status = 0;
  }
}

// ---------------------------------------------------------------- K2 PCA  (pca_score :179-183)
// balanced columns (drop_missing_col :167-170).  grid (B), single thread.
__global__ void k_balanced_cols(const int* col_n, int T, int N, int* bal_idx, int* nbal) {
  if (DFM_TID != 0) return;
  int b = DFM_BX, n = 0;
  for (int i = 0; i < N; ++i) if (col_n[(size_t)b * N + i] == T) bal_idx[(size_t)b * N + n++] = i;
  nbal[b] = n;
}
__global__ void k_all_cols(int N, int* bal_idx, int* nbal) {
  int b = DFM_BX;
  for (int i = DFM_TID; i < N; i += DFM_NT) bal_idx[(size_t)b * N + i] = i;
  if (DFM_TID == 0) nbal[b] = N;
}

// Gram of the balanced block: mode 0 (nbal <= T): G = Xb'Xb (nbal x nbal); mode 1: G = Xb Xb' (T x T).
// G stored dense with leading dimension n = min(nbal, T).
// On the FP64 tensor path: one WARP per 16 x 16 block of the lower triangle (2 x 2 DMMA tiles: two A and two
// B fragments per four DMMA.8x8x4), fragments straight from global memory -- a panel (<= 1 MB) is L2 resident and every
// 32-byte sector a fragment load touches is used completely; the reduction runs over T (mode 0) or over the balanced
// columns (mode 1).  grid (ceil(nblocks / 8), B), 256 threads, nblocks = nb16 (nb16 + 1) / 2 with nb16 = ceil(nmax / 16).
__global__ void k_gram_tc(const double* __restrict__ Xs, int T, int N, const int* __restrict__ bal_idx,
                          const int* __restrict__ nbal, double* __restrict__ G, int nmax) {
#ifndef DFM_EMU
  const int b = DFM_BY;
  const int nb = nbal[b];
  const int mode = (nb <= T) ? 0 : 1;
  const int n = mode ? T : nb, K = mode ? nb : T;
  const int nb16 = (n + 15) >> 4;
  const int blk = DFM_BX * DFM_NWARP + DFM_WARP;
  if (blk >= nb16 * (nb16 + 1) / 2) return;
  int bi = (int)((sqrt(8.0 * blk + 1.0) - 1.0) * 0.5);
  while ((bi + 1) * (bi + 2) / 2 <= blk) ++bi;
  while (bi * (bi + 1) / 2 > blk) --bi;
  const int bj = blk - bi * (bi + 1) / 2;                 // bj <= bi
  const double* X = Xs + (size_t)b * T * N;
  const int* idx = bal_idx + (size_t)b * N;
  double* g = G + (size_t)b * nmax * nmax;
  const int lr = DFM_LANE >> 2, lc = DFM_LANE & 3;
  const int r0 = bi * 16 + lr, r1 = r0 + 8, c0 = bj * 16 + lr, c1 = c0 + 8;
  double d00[2] = {0.0, 0.0}, d01[2] = {0.0, 0.0}, d10[2] = {0.0, 0.0}, d11[2] = {0.0, 0.0};
#define GR_DMMA(d_, a_, b_) asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n" : "+d"((d_)[0]), "+d"((d_)[1]) : "d"(a_), "d"(b_))
  if (mode == 0) {
    const double* pa0 = (r0 < n) ? X + (size_t)T * idx[r0] : nullptr; const double* pa1 = (r1 < n) ? X + (size_t)T * idx[r1] : nullptr;
    const double* pb0 = (c0 < n) ? X + (size_t)T * idx[c0] : nullptr; const double* pb1 = (c1 < n) ? X + (size_t)T * idx[c1] : nullptr;
#pragma unroll 4
    for (int l0 = 0; l0 < K; l0 += 4) {
      const int l = l0 + lc;
      const bool lok = l < K;
      const double a0 = (pa0 && lok) ? pa0[l] : 0.0, a1 = (pa1 && lok) ? pa1[l] : 0.0;
      const double b0 = (pb0 && lok) ? pb0[l] : 0.0, b1 = (pb1 && lok) ? pb1[l] : 0.0;
      GR_DMMA(d00, a0, b0); GR_DMMA(d01, a0, b1); GR_DMMA(d10, a1, b0); GR_DMMA(d11, a1, b1);
    }
  } else {
#pragma unroll 4
    for (int l0 = 0; l0 < K; l0 += 4) {
      const int l = l0 + lc;
      const double* col = (l < K) ? X + (size_t)T * idx[l] : nullptr;
      const double a0 = (col && r0 < n) ? col[r0] : 0.0, a1 = (col && r1 < n) ? col[r1] : 0.0;
      const double b0 = (col && c0 < n) ? col[c0] : 0.0, b1 = (col && c1 < n) ? col[c1] : 0.0;
      GR_DMMA(d00, a0, b0); GR_DMMA(d01, a0, b1); GR_DMMA(d10, a1, b0); GR_DMMA(d11, a1, b1);
    }
  }
#undef GR_DMMA
  // element (row, col) of tile (ti, tj): row = bi*16 + 8 ti + lr, col = bj*16 + 8 tj + 2 lc (+1); lower triangle, mirrored
  auto put = [&](int row, int col, double v) { if (row < n && col < n && row >= col) { g[row + (size_t)n * col] = v; g[col + (size_t)n * row] = v; } };
  const int cc = bj * 16 + 2 * lc;
  put(r0, cc, d00[0]); put(r0, cc + 1, d00[1]); put(r0, cc + 8, d01[0]); put(r0, cc + 9, d01[1]);
  put(r1, cc, d10[0]); put(r1, cc + 1, d10[1]); put(r1, cc + 8, d11[0]); put(r1, cc + 9, d11[1]);
#else
  // emulation: plain sums (same entries)
  int b = DFM_BY;
  int nb = nbal[b];
  int mode = (nb <= T) ? 0 : 1;
  int n = mode ? T : nb;
  if (DFM_BX != 0) return;
  const double* X = Xs + (size_t)b * T * N;
  const int* idx = bal_idx + (size_t)b * N;
  double* g = G + (size_t)b * nmax * nmax;
  for (int c = 0; c < n; ++c)
    for (int a = c; a < n; ++a) {
      double s = 0.0;
      if (mode == 0) { const double* xa = X + (size_t)idx[a] * T; const double* xc = X + (size_t)idx[c] * T; for (int t = 0; t < T; ++t) s += xa[t] * xc[t]; }
      else for (int j = 0; j < nb; ++j) { const double* col = X + (size_t)idx[j] * T; s += col[a] * col[c]; }
      g[a + (size_t)n * c] = s; g[c + (size_t)n * a] = s;
    }
#endif
}

// Cyclic Jacobi eigen-solver core (round-robin parallel ordering) on an n x n symmetric matrix G with
// leading dimension n (shared or global memory).  G is destroyed (diagonal = eigenvalues); V (n x n,
// ld n) receives the eigenvectors in its columns.  cs: 2 (n + 2) doubles, red: 40 doubles of shared scratch.
// Block-cooperative; returns the number of sweeps.  Per round: the m/2 disjoint pairs and their rotations are tabulated
// once (reciprocals / reciprocal square roots from the hardware seed), then applied with warp = pair, lane = column --
// no index arithmetic in the element loops, three barriers per round.
__device__ inline int jacobi_core(double* G, double* V, int n, double* cs, double* red, int max_sweeps) {
  int m = (n + 1) & ~1;                  // even number of players
  int* pq = (int*)(cs + m + 2);          // [m/2][2] pair table of the round
  for (int e = DFM_TID; e < n * n; e += DFM_NT) { int i = e % n, j = e / n; V[i + (size_t)n * j] = (i == j) ? 1.0 : 0.0; }
  DFM_SYNC();
  int sweep = 0;
  for (; sweep < max_sweeps; ++sweep) {
    double off = 0.0, dg = 0.0;
    for (int j = DFM_WARP; j < n; j += DFM_NWARP)
      for (int i = DFM_LANE; i < n; i += DFM_WSZ) {
        double v = G[i + (size_t)n * j];
        if (i > j) off += v * v; else if (i == j) dg += v * v;
      }
    off = block_sum(off, red); dg = block_sum(dg, red);
    if (off <= 1e-30 * dg) break;         // off-diagonal norm <= 1e-15 of the diagonal norm
    for (int s = 0; s < m - 1; ++s) {
      // phase 1: pairs and rotation angles of this round
      for (int i = DFM_TID; i < m / 2; i += DFM_NT) {
        int j1 = i, j2 = m - 1 - i;
        int p = (j1 == 0) ? 0 : ((j1 - 1 + s) % (m - 1)) + 1;
        int q = (j2 == 0) ? 0 : ((j2 - 1 + s) % (m - 1)) + 1;
        if (p > q) { int t_ = p; p = q; q = t_; }
        double c = 1.0, sn = 0.0;
        if (q < n) {
          double app = G[p + (size_t)n * p], aqq = G[q + (size_t)n * q], apq = G[p + (size_t)n * q];
          if (fabs(apq) > 1e-300 && fabs(apq) * fabs(apq) > 1e-36 * fabs(app * aqq)) {
            double tau = (aqq - app) * 0.5 * fast_rcp(apq);
            double h = 1.0 + tau * tau;
            double t = ((tau >= 0.0) ? 1.0 : -1.0) * fast_rcp(fabs(tau) + h * fast_rsqrt(h));
            c = fast_rsqrt(1.0 + t * t); sn = t * c;
          }
        } else q = -1;
        cs[2 * i] = c; cs[2 * i + 1] = sn; pq[2 * i] = p; pq[2 * i + 1] = q;
      }
      DFM_SYNC();
      // phase 2: G <- J' G  (rows p, q)
      for (int i = DFM_WARP; i < m / 2; i += DFM_NWARP) {
        const int p = pq[2 * i], q = pq[2 * i + 1];
        if (q < 0) continue;
        const double c = cs[2 * i], sn = cs[2 * i + 1];
        for (int j = DFM_LANE; j < n; j += DFM_WSZ) {
          double gp = G[p + (size_t)n * j], gq = G[q + (size_t)n * j];
          G[p + (size_t)n * j] = c * gp - sn * gq;
          G[q + (size_t)n * j] = sn * gp + c * gq;
        }
      }
      DFM_SYNC();
      // phase 3: G <- G J, V <- V J  (columns p, q)
      for (int i = DFM_WARP; i < m / 2; i += DFM_NWARP) {
        const int p = pq[2 * i], q = pq[2 * i + 1];
        if (q < 0) continue;
        const double c = cs[2 * i], sn = cs[2 * i + 1];
        for (int j = DFM_LANE; j < n; j += DFM_WSZ) {
          double gp = G[j + (size_t)n * p], gq = G[j + (size_t)n * q];
          G[j + (size_t)n * p] = c * gp - sn * gq;
          G[j + (size_t)n * q] = sn * gp + c * gq;
          double vp = V[j + (size_t)n * p], vq = V[j + (size_t)n * q];
          V[j + (size_t)n * p] = c * vp - sn * vq;
          V[j + (size_t)n * q] = sn * vp + c * vq;
        }
      }
      DFM_SYNC();
    }
  }
  return sweep;
}

// Direct Jacobi on the Gram matrix (small n <= 64): the matrix and the eigenvector matrix live in shared memory for the
// sweeps (copy in, rotate, copy out).  grid (B), one block per panel; shared 2 n^2 + 2 (n + 2) + 48 doubles.
__global__ void k_jacobi(double* __restrict__ Gall, double* __restrict__ Vall, const int* __restrict__ nbal,
                         int T, int nmax, int max_sweeps, int* __restrict__ sweeps_out) {
  DFM_SMEM(sm);
  int b = DFM_BX;
  int nb = nbal[b];
  int n = (nb <= T) ? nb : T;
  double* G = Gall + (size_t)b * nmax * nmax;
  double* V = Vall + (size_t)b * nmax * nmax;
  int m = (n + 1) & ~1;
  double* Gs = sm; double* Vs = Gs + (size_t)n * n; double* cs = Vs + (size_t)n * n;
  for (int e = DFM_TID; e < n * n; e += DFM_NT) Gs[e] = G[e];
  DFM_SYNC();
  int sw = jacobi_core(Gs, Vs, n, cs, cs + 2 * (m + 2), max_sweeps);
  DFM_SYNC();
  for (int e = DFM_TID; e < n * n; e += DFM_NT) { G[e] = Gs[e]; V[e] = Vs[e]; }
  if (DFM_TID == 0 && sweeps_out) sweeps_out[b] = sw;
}

// Top-m eigenpairs of the Gram matrix by block subspace iteration with Rayleigh-Ritz (n > 64):
//   V <- orth(G V) (CholQR2), H = V'GV (m x m), Jacobi on H in shared memory, V <- V W,
// until the residuals ||G v_i - theta_i v_i|| of the leading r pairs drop below tol * theta_1.
// Results are left in the layout k_pca_finish expects: eigenvalues on the diagonal of G (entries
// m..n-1 set to -1e300), Ritz vectors in the first m columns of V (ld n).  grid (B), one block.
// Y: global scratch n x m per panel.  shared: 3 m^2 + m + 64 doubles.
__global__ void k_subspace_eig(double* __restrict__ Gall, double* __restrict__ Vall, double* __restrict__ Yall,
                               const int* __restrict__ nbal, int T, int nmax, int r, int mmax, int maxit, double tol,
                               int* __restrict__ iters_out) {
  DFM_SMEM(sm);
  int b = DFM_BX;
  int nb = nbal[b];
  int n = (nb <= T) ? nb : T;
  int m = (mmax < n) ? mmax : n;
  double* G = Gall + (size_t)b * nmax * nmax;
  double* V = Vall + (size_t)b * nmax * nmax;           // n x m in the first m columns
  double* Y = Yall + (size_t)b * nmax * mmax;           // n x m
  double* H = sm; double* W = H + m * m; double* S = W + m * m; double* cs = S + m * m; double* red = cs + 2 * (m + 2);
  int* info = (int*)(red + 40);
  double* theta = red + 44;                              // m
  if (DFM_TID == 0) *info = 0;
  // deterministic start: V[i][j] = hash-based pseudo-random in (-1, 1)
  for (int e = DFM_TID; e < n * m; e += DFM_NT) {
    unsigned h = (unsigned)e * 2654435761u + 12345u; h ^= h >> 15; h *= 2246822519u; h ^= h >> 13; h *= 3266489917u; h ^= h >> 16;
    V[e] = (double)(h & 0xffffff) / 8388608.0 - 1.0;
  }
  DFM_SYNC();
  int it = 0;
  double res = 1.0;
  for (; it < maxit; ++it) {
    // ---- orthonormalise V (CholQR, twice): S = V'V = L L', V <- V L^-T
    for (int pass = 0; pass < 2; ++pass) {
      for (int e = DFM_TID; e < m * m; e += DFM_NT) {
        int a = e % m, c = e / m;
        if (a < c) continue;
        double s = 0.0;
        for (int i = 0; i < n; ++i) s += V[i + (size_t)n * a] * V[i + (size_t)n * c];
        S[a + m * c] = s; S[c + m * a] = s;
      }
      DFM_SYNC();
      bm_chol(S, m, m, info);
      for (int i = DFM_TID; i < n; i += DFM_NT) {        // row i: x L' = v  (forward substitution over columns)
        for (int c = 0; c < m; ++c) {
          double s = V[i + (size_t)n * c];
          for (int l = 0; l < c; ++l) s -= S[c + m * l] * V[i + (size_t)n * l];
          V[i + (size_t)n * c] = s / S[c + m * c];
        }
      }
      DFM_SYNC();
    }
    // ---- Y = G V
    for (int e = DFM_TID; e < n * m; e += DFM_NT) {
      int i = e % n, j = e / n;
      double s = 0.0;
      for (int l = 0; l < n; ++l) s += G[i + (size_t)n * l] * V[l + (size_t)n * j];
      Y[e] = s;
    }
    DFM_SYNC();
    // ---- Rayleigh-Ritz: H = V'Y, eigen-decomposition in shared memory, rotate V and Y
    for (int e = DFM_TID; e < m * m; e += DFM_NT) {
      int a = e % m, c = e / m;
      if (a < c) continue;
      double s = 0.0;
      for (int i = 0; i < n; ++i) s += V[i + (size_t)n * a] * Y[i + (size_t)n * c];
      H[a + m * c] = s; H[c + m * a] = s;
    }
    DFM_SYNC();
    jacobi_core(H, W, m, cs, red, 40);
    // order the Ritz values (descending) -> theta, permutation kept in cs (as doubles)
    if (DFM_TID == 0) {
      for (int j = 0; j < m; ++j) {
        int best = -1; double bv = -1e300;
        for (int i = 0; i < m; ++i) { bool used = false; for (int l = 0; l < j; ++l) if ((int)cs[l] == i) used = true;
          if (!used && H[i + m * i] > bv) { bv = H[i + m * i]; best = i; } }
        cs[j] = (double)best; theta[j] = bv;
      }
    }
    DFM_SYNC();
    // V <- V W[:, perm], Y <- Y W[:, perm]   (row by row, m x m product per row, in place via registers is too
    // big: use S as per-thread-row staging is not possible either -> two passes through S rows in chunks)
    for (int i = DFM_TID; i < n; i += DFM_NT) {
      // rotate row i of V then of Y using a small local buffer in registers (m <= 64)
      double rowv[64];
      for (int c = 0; c < m; ++c) rowv[c] = V[i + (size_t)n * c];
      for (int j = 0; j < m; ++j) { int pj = (int)cs[j]; double s = 0.0; for (int c = 0; c < m; ++c) s += rowv[c] * W[c + m * pj]; V[i + (size_t)n * j] = s; }
      for (int c = 0; c < m; ++c) rowv[c] = Y[i + (size_t)n * c];
      for (int j = 0; j < m; ++j) { int pj = (int)cs[j]; double s = 0.0; for (int c = 0; c < m; ++c) s += rowv[c] * W[c + m * pj]; Y[i + (size_t)n * j] = s; }
    }
    DFM_SYNC();
    // ---- residuals of the leading r pairs
    double rmax = 0.0;
    for (int j = 0; j < r; ++j) {
      double s = 0.0;
      for (int i = DFM_TID; i < n; i += DFM_NT) { double d = Y[i + (size_t)n * j] - theta[j] * V[i + (size_t)n * j]; s += d * d; }
      s = block_sum(s, red);
      rmax = fmax(rmax, sqrt(s));
    }
    res = rmax / fabs(theta[0]);
    if (res <= tol) { ++it; break; }
    // next iterate: V <- G^q V (q = 3 products per orthonormalisation + Rayleigh-Ritz cycle: the cycle -- CholQR2 and a
    // Jacobi eigen-solve of the m x m projected matrix -- costs far more than a product, and the error of the wanted
    // pairs contracts by (lambda_{m+1} / lambda_r)^q per cycle; Y = G V of the rotated basis is already there)
    for (int e = DFM_TID; e < n * m; e += DFM_NT) V[e] = Y[e];
    DFM_SYNC();
    for (int q_ = 1; q_ < 3; ++q_) {
      for (int e = DFM_TID; e < n * m; e += DFM_NT) {
        int i = e % n, j = e / n;
        double s = 0.0;
        for (int l = 0; l < n; ++l) s += G[i + (size_t)n * l] * V[l + (size_t)n * j];
        Y[e] = s;
      }
      DFM_SYNC();
      // rescale the columns (plain power steps grow like lambda^q): keeps the Gram matrix of CholQR well scaled
      for (int j = 0; j < m; ++j) {
        double s = 0.0;
        for (int i = DFM_TID; i < n; i += DFM_NT) s += Y[i + (size_t)n * j] * Y[i + (size_t)n * j];
        s = block_sum(s, red);
        const double sc_ = (s > 0.0) ? 1.0 / sqrt(s) : 1.0;
        for (int i = DFM_TID; i < n; i += DFM_NT) V[i + (size_t)n * j] = Y[i + (size_t)n * j] * sc_;
      }
      DFM_SYNC();
    }
  }
  // ---- leave results where k_pca_finish looks for them
  for (int i = DFM_TID; i < n; i += DFM_NT) G[i + (size_t)n * i] = (i < m) ? theta[i] : -1e300;
  if (DFM_TID == 0 && iters_out) iters_out[b] = (res <= tol) ? it : -it;
}

// Y (n x m, ld ldv, shared) = G (n x n, ld n, global: L2 resident) * V (n x m, ld ldv, shared) on the tensor path.  One warp per
// 8-row block of Y: its A fragments (rows of G) are read straight from L2, EIGHT k-steps ahead of the DMMAs (a fragment
// load from L2 has a long latency: two in flight, as in the generic tile product, leave the loop latency bound), and each
// fragment feeds all ceil(m / 8) <= 6 column tiles, whose B fragments come conflict-free from the shared iterate.
__device__ __forceinline__ void gv_product(const double* __restrict__ G, int n, const double* V, double* Y, int ldv, int m);
// general form: Y (rows x m, ld ldy) = A (rows x K, element (i, l) at A[i + lda * l], global) * V (K x m, ld ldv, shared)
__device__ __forceinline__ void av_product(const double* __restrict__ G, int rows, int K, size_t lda, const double* V, int ldv, double* Y,
                                           size_t ldy, int m) {
#ifndef DFM_EMU
  const int lr = DFM_LANE >> 2, lc = DFM_LANE & 3;
  const int n = K;
  const int nrb = (rows + 7) >> 3, nct = (m + 7) >> 3;
  for (int rb = DFM_WARP; rb < nrb; rb += DFM_NWARP) {
    const int row = rb * 8 + lr;
    const bool rok = row < rows;
    const double* gp = G + (rok ? row : 0);
    double d[6][2];
#pragma unroll
    for (int ct = 0; ct < 6; ++ct) { d[ct][0] = 0.0; d[ct][1] = 0.0; }
    for (int l0 = 0; l0 < n; l0 += 32) {
      double a[8];
#pragma unroll
      for (int q = 0; q < 8; ++q) { const int l = l0 + 4 * q + lc; a[q] = (rok && l < n) ? gp[lda * l] : 0.0; }
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const int l = l0 + 4 * q + lc;
        const bool lok = l < n;
#pragma unroll
        for (int ct = 0; ct < 6; ++ct) {
          if (ct < nct) {
            const int col = ct * 8 + lr;
            const double bz = (lok && col < m) ? V[l + (size_t)ldv * col] : 0.0;
            EM_DMMA(d[ct], a[q], bz);
          }
        }
      }
    }
    if (rok) {
#pragma unroll
      for (int ct = 0; ct < 6; ++ct) {
        const int col = ct * 8 + 2 * lc;
        if (col < m) Y[row + ldy * col] = d[ct][0];
        if (col + 1 < m) Y[row + ldy * (col + 1)] = d[ct][1];
      }
    }
  }
#else
  for (int j = 0; j < m; ++j)
    for (int i = 0; i < rows; ++i) {
      double v = 0.0;
      for (int l = 0; l < K; ++l) v += G[i + lda * l] * V[l + (size_t)ldv * j];
      Y[i + ldy * j] = v;
    }
#endif
  DFM_SYNC();
}
__device__ __forceinline__ void gv_product(const double* __restrict__ G, int n, const double* V, double* Y, int ldv, int m) {
  av_product(G, n, n, (size_t)n, V, ldv, Y, (size_t)ldv, m);
}

// Shared-memory / tensor-core variant of k_subspace_eig for panels whose iterate fits shared memory (2 n m doubles):
// the n x m iterate V and the product Y = G V stay in shared memory, every product (G V, V'V, V'Y, V W) is a DMMA tile
// product (wt_gemm; G is read from L2), CholQR uses the block-cooperative Cholesky + transposed solves, and the
// Rayleigh-Ritz step (Jacobi on the m x m projected matrix: the expensive, serial part) runs after the third cycle of
// q = 3 products and then every second cycle -- between them the subspace just keeps converging under orth(G^3 V).  Same results layout as
// k_subspace_eig.  grid (B), 256 threads; shared 2 n ldv... see subspace2_smem_doubles.
__host__ __device__ inline size_t subspace2_smem_doubles(int n, int m) {
  return 2 * (size_t)em_lds(n) * m + 3 * (size_t)m * m + 2 * (m + 2) + 64 + 2 * m + 64;
}
#ifdef DFM_EMU
#define SUB2_BOUNDS
#else
#define SUB2_BOUNDS __launch_bounds__(256, 2)
#endif
__global__ void SUB2_BOUNDS k_subspace_eig2(double* __restrict__ Gall, double* __restrict__ Vall, const int* __restrict__ nbal, int T,
                                int nmax, int r, int mmax, int maxit, double tol, int* __restrict__ iters_out) {
  DFM_SMEM(sm);
  int b = DFM_BX;
  int nb = nbal[b];
  int n = (nb <= T) ? nb : T;
  int m = (mmax < n) ? mmax : n;
  const int ldv = em_lds(n);
  const double* G = Gall + (size_t)b * nmax * nmax;
  double* Vg = Vall + (size_t)b * nmax * nmax;          // result: n x m in the first m columns (ld n)
  double* Gd = Gall + (size_t)b * nmax * nmax;
  double* V = sm; double* Y = V + (size_t)ldv * m;
  double* H = Y + (size_t)ldv * m; double* W = H + m * m; double* S = W + m * m; double* cs = S + m * m;
  double* red = cs + 2 * (m + 2);                        // 40
  int* info = (int*)(red + 40);
  double* theta = red + 44;                              // m
  double* dinv = theta + m;                              // m
  double* perm = dinv + m;                               // m (as doubles)
  if (DFM_TID == 0) *info = 0;
  // deterministic start: V[i][j] = hash-based pseudo-random in (-1, 1)   (same start as k_subspace_eig)
  for (int e = DFM_TID; e < n * m; e += DFM_NT) {
    unsigned h = (unsigned)e * 2654435761u + 12345u; h ^= h >> 15; h *= 2246822519u; h ^= h >> 13; h *= 3266489917u; h ^= h >> 16;
    V[(e % n) + (size_t)ldv * (e / n)] = (double)(h & 0xffffff) / 8388608.0 - 1.0;
  }
  DFM_SYNC();
  int it = 0;
  double res = 1.0;
  for (; it < maxit; ++it) {
    // ---- orthonormalise V (CholQR, twice): S = V'V = L L', V <- V L^-T  (row-wise transposed solve)
    for (int pass = 0; pass < 2; ++pass) {
      wt_gemm(V, ldv, 1, V, ldv, 1, m, m, n, [&](int a, int c, double v) { S[a + m * c] = v; });
      DFM_SYNC();
      bm_symmetrize(S, m, m);
      bc_chol(S, m, m, dinv, info);
      bt_trsm_lower(S, m, m, dinv, V, ldv, n);
    }
    // Rayleigh-Ritz + convergence test: first after three cycles (9 products: a well separated factor spectrum has converged
    // by then), afterwards every second cycle -- the Jacobi solve of the projected matrix is the expensive, serial part
    const bool rr = (it >= 2 && ((it - 2) & 1) == 0) || it + 1 >= maxit;
    // ---- Y = G V
    gv_product(G, n, V, Y, ldv, m);
    if (rr) {
      wt_gemm(V, ldv, 1, Y, ldv, 1, m, m, n, [&](int a, int c, double v) { H[a + m * c] = v; });
      DFM_SYNC();
      bm_symmetrize(H, m, m);
      jacobi_core(H, W, m, cs, red, 40);
      if (DFM_TID == 0) {                                 // Ritz values in descending order (selection with used flags in cs: O(m^2))
        for (int i = 0; i < m; ++i) cs[i] = 0.0;
        for (int j = 0; j < m; ++j) {
          int best = -1; double bv = -1e300;
          for (int i = 0; i < m; ++i) { const double hv = H[i + m * i]; if (cs[i] == 0.0 && hv > bv) { bv = hv; best = i; } }
          perm[j] = (double)best; theta[j] = bv; cs[best] = 1.0;
        }
      }
      DFM_SYNC();
      for (int e = DFM_TID; e < m * m; e += DFM_NT) { const int c = e % m, j = e / m; S[e] = W[c + m * (int)perm[j]]; }   // permuted rotation
      DFM_SYNC();
      // rotate both V and Y into the Ritz basis: through H/W-sized scratch is impossible (n x m): rotate V into Y's place
      // after Y has been rotated in place row by row?  -- simpler and cheap on the tensor path: V' = V S (into scratch = Y
      // is busy), so: first Y <- Y S via a second buffer = V is busy too.  Use the identity Y S = G (V S): rotate V into Y,
      // swap, and recompute Y = G V.
      wt_gemm(V, 1, ldv, S, m, 1, n, m, m, [&](int i, int j, double v) { Y[i + (size_t)ldv * j] = v; });
      DFM_SYNC();
      { double* sw = V; V = Y; Y = sw; }
      gv_product(G, n, V, Y, ldv, m);
      // ---- residuals of the leading r pairs
      double rmax = 0.0;
      for (int j = 0; j < r; ++j) {
        double s_ = 0.0;
        for (int i = DFM_TID; i < n; i += DFM_NT) { double d = Y[i + (size_t)ldv * j] - theta[j] * V[i + (size_t)ldv * j]; s_ += d * d; }
        s_ = block_sum(s_, red);
        rmax = fmax(rmax, sqrt(s_));
      }
      res = rmax / fabs(theta[0]);
      if (res <= tol) { ++it; break; }
    }
    // next iterate: V <- normalised G^3 V (Y = G V is there)
    for (int q_ = 0; q_ < 3; ++q_) {
      if (q_ > 0) {
        gv_product(G, n, V, Y, ldv, m);
      }
      // rescale the columns (plain power steps grow like lambda^q): keeps the Gram matrix of CholQR well scaled
      for (int j = DFM_WARP; j < m; j += DFM_NWARP) {
        double s_ = 0.0;
        for (int i = DFM_LANE; i < n; i += DFM_WSZ) s_ += Y[i + (size_t)ldv * j] * Y[i + (size_t)ldv * j];
#ifndef DFM_EMU
        for (int o = 16; o > 0; o >>= 1) s_ += __shfl_xor_sync(0xffffffffu, s_, o);
#endif
        const double sc_ = (s_ > 0.0) ? 1.0 / sqrt(s_) : 1.0;
        for (int i = DFM_LANE; i < n; i += DFM_WSZ) V[i + (size_t)ldv * j] = Y[i + (size_t)ldv * j] * sc_;
      }
      DFM_SYNC();
    }
  }
  // ---- leave results where k_pca_finish looks for them
  for (int e = DFM_TID; e < n * m; e += DFM_NT) Vg[e] = V[(e % n) + (size_t)ldv * (e / n)];
  DFM_SYNC();
  for (int i = DFM_TID; i < n; i += DFM_NT) Gd[i + (size_t)n * i] = (i < m) ? theta[i] : -1e300;
  if (DFM_TID == 0 && iters_out) iters_out[b] = (res <= tol) ? it : -it;
}

// Pick the r largest eigenpairs and form scores.  grid (B), one block.
// mode 0: score_j = Xb v_j ; mode 1: score_j = u_j * sqrt(lambda_j).  Sign: the entry of largest
// magnitude of the right singular vector v_j is made positive.
__global__ void k_pca_finish(const double* __restrict__ Xs, int T, int N, const int* __restrict__ bal_idx,
                             const int* __restrict__ nbal, const double* __restrict__ Gall,
                             const double* __restrict__ Vall, int nmax, int r, double* __restrict__ score,
                             int* __restrict__ status, AlsState* st, int fast_smem = 0) {
  DFM_SMEM(sm);
  int b = DFM_BX;
  int nb = nbal[b];
  int mode = (nb <= T) ? 0 : 1;
  int n = mode ? T : nb;
  const double* X = Xs + (size_t)b * T * N;
  const int* idx = bal_idx + (size_t)b * N;
  const double* G = Gall + (size_t)b * nmax * nmax;
  const double* V = Vall + (size_t)b * nmax * nmax;
  double* sc = score + (size_t)b * T * r;
  int* order = (int*)sm;                 // r ints
  double* red = sm + ((r + 1) / 2 + 1);  // 33+
  double* vtmp = red + 40;               // nb doubles (mode 1)
  if (n < r) { if (DFM_TID == 0) { if (status) status[b] = 2; if (st) { st[b].status = 2; st[b].done = 1; } } return; }
  if (DFM_WARP == 0) {                   // selection of the r largest diagonal entries: one warp, argmax by shuffles per pick
    for (int j = 0; j < r; ++j) {            // (ties: the smallest index, as a serial scan with `>` gives)
      int best = n; double bv = -1e300;
      for (int i = DFM_LANE; i < n; i += DFM_WSZ) {
        bool used = false;
        for (int l = 0; l < j; ++l) if (order[l] == i) used = true;
        double v = G[i + (size_t)n * i];
        if (!used && (v > bv || (v == bv && i < best))) { bv = v; best = i; }
      }
#ifndef DFM_EMU
      for (int o = 16; o > 0; o >>= 1) {
        const double ov = __shfl_xor_sync(0xffffffffu, bv, o); const int oi = __shfl_xor_sync(0xffffffffu, best, o);
        if (ov > bv || (ov == bv && oi < best)) { bv = ov; best = oi; }
      }
#endif
      if (DFM_LANE == 0) order[j] = best;
      DFM_WSYNC();
    }
  }
  DFM_SYNC();
  if (mode == 0 && nb == N && r <= 48 && fast_smem) {
    // every column is balanced (idx = identity): scores = X Vr on the tensor path, Vr = the r selected eigenvectors with
    // their signs, staged in shared memory
    double* Vr = vtmp;                                   // n x r, ld em_lds(n)
    const int ldr = em_lds(n);
    for (int j = DFM_WARP; j < r; j += DFM_NWARP) {
      const double* v = V + (size_t)n * order[j];
      double best = 0.0, sg = 1.0; int bi = n;           // largest |entry|, first index on ties (as the scalar path)
      for (int i = DFM_LANE; i < n; i += DFM_WSZ) if (fabs(v[i]) > best) { best = fabs(v[i]); sg = (v[i] < 0) ? -1.0 : 1.0; bi = i; }
#ifndef DFM_EMU
      for (int o = 16; o > 0; o >>= 1) {
        const double ob = __shfl_xor_sync(0xffffffffu, best, o), os = __shfl_xor_sync(0xffffffffu, sg, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ob > best || (ob == best && oi < bi)) { best = ob; sg = os; bi = oi; }
      }
#endif
      for (int i = DFM_LANE; i < n; i += DFM_WSZ) Vr[i + (size_t)ldr * j] = sg * v[i];
    }
    DFM_SYNC();
    av_product(X, T, n, (size_t)T, Vr, ldr, sc, (size_t)T, r);
    return;
  }
  for (int j = 0; j < r; ++j) {
    const double* v = V + (size_t)n * order[j];
    if (mode == 0) {
      // sign from v itself (thread 0; n is small)
      if (DFM_TID == 0) {
        double best = 0.0, sg = 1.0;
        for (int i = 0; i < n; ++i) if (fabs(v[i]) > best) { best = fabs(v[i]); sg = (v[i] < 0) ? -1.0 : 1.0; }
        red[36] = sg;
      }
      DFM_SYNC();
      double sg = red[36];
      for (int t = DFM_TID; t < T; t += DFM_NT) {
        double s = 0.0;
        for (int i = 0; i < n; ++i) s += X[t + (size_t)T * idx[i]] * v[i];
        sc[t + (size_t)T * j] = sg * s;
      }
      DFM_SYNC();
    } else {
      double lam = G[order[j] + (size_t)n * order[j]];
      double sig = sqrt(lam > 0 ? lam : 0.0);
      // right singular vector (up to scale): w = Xb' u
      for (int i = DFM_TID; i < nb; i += DFM_NT) {
        const double* col = X + (size_t)idx[i] * T;
        double s = 0.0;
        for (int t = 0; t < T; ++t) s += col[t] * v[t];
        vtmp[i] = s;
      }
      DFM_SYNC();
      if (DFM_TID == 0) {
        double best = 0.0, sg = 1.0;
        for (int i = 0; i < nb; ++i) if (fabs(vtmp[i]) > best) { best = fabs(vtmp[i]); sg = (vtmp[i] < 0) ? -1.0 : 1.0; }
        red[36] = sg;
      }
      DFM_SYNC();
      double sg = red[36];
      for (int t = DFM_TID; t < T; t += DFM_NT) sc[t + (size_t)T * j] = sg * sig * v[t];
      DFM_SYNC();
    }
  }
}

// ---------------------------------------------------------------- K3 ALS sweep  (:352-370)
// out (r x r) = M'M over rows whose first entry is not NaN.  M is nrow x r, ld nrow.  grid (B).
__global__ void k_gram_small(const double* __restrict__ Mall, int nrow, int r, double* __restrict__ out,
                             const AlsState* st) {
  int b = DFM_BX;
  if (st && st[b].done) return;
  const double* M = Mall + (size_t)b * nrow * r;
  double* o = out + (size_t)b * r * r;
  for (int e = DFM_TID; e < r * r; e += DFM_NT) {
    int a = e % r, c = e / r;
    if (a < c) continue;
    double s = 0.0;
    for (int t = 0; t < nrow; ++t) { double m0 = M[t]; if (!is_nan(m0)) s += M[t + (size_t)nrow * a] * M[t + (size_t)nrow * c]; }
    o[a + r * c] = s; o[c + r * a] = s;
  }
}

// Lambda-step (:355-362): one block per series.  mode 0: write Lam (NaN if < nt_min obs), apply the
// :factor constraint (:1125-1141);  mode 1: R2 of the per-series regression (:372-380);
// mode 2: EM initialisation: Lam and R_i = ssr_i / T_i.
// FtF = F'F over ALL rows (used only by the constraint, which passes the full f: :360).
__global__ void k_als_lambda(const double* __restrict__ Xs, const double* __restrict__ Fall, int T, int N, int r,
                             int nt_min, int mode, double* __restrict__ Lam, double* __restrict__ out2,
                             const double* __restrict__ FtF, int n_constr, const int* __restrict__ c_index,
                             const double* __restrict__ c_R, const double* __restrict__ c_r,
                             const double* __restrict__ xstd, AlsState* st, const int* __restrict__ only_missing = nullptr) {
  DFM_SMEM(sm);
  int i = DFM_BX, b = DFM_BY;
  if (st && st[b].done && mode == 0) return;
  if (only_missing && !only_missing[b]) return;          // (EM initialisation: balanced panels take k_emb_mstep)
  const double* x = Xs + ((size_t)b * N + i) * T;
  const double* F = Fall + (size_t)b * T * r;
  int np = r * (r + 1) / 2;
  double* A = sm;                 // packed np
  double* c = A + np;             // r
  double* sc = c + r;             // [0]=cnt [1]=sxx [2]=sx
  double* wk = sc + 4;            // constraint workspace
  int nwork = np + r + 3;
  for (int e = DFM_TID; e < nwork; e += DFM_NT) {
    double s = 0.0;
    if (e < np) {
      int a = 0; while ((a + 1) * (a + 2) / 2 <= e) ++a;
      int cc = e - a * (a + 1) / 2;
      const double* fa = F + (size_t)T * a; const double* fc = F + (size_t)T * cc;
      for (int t = 0; t < T; ++t) if (!is_nan(x[t])) s += fa[t] * fc[t];
      A[e] = s;
    } else if (e < np + r) {
      const double* fa = F + (size_t)T * (e - np);
      for (int t = 0; t < T; ++t) { double v = x[t]; if (!is_nan(v)) s += v * fa[t]; }
      c[e - np] = s;
    } else if (e == np + r) {
      for (int t = 0; t < T; ++t) if (!is_nan(x[t])) s += 1.0;
      sc[0] = s;
    } else if (e == np + r + 1) {
      for (int t = 0; t < T; ++t) { double v = x[t]; if (!is_nan(v)) s += v * v; }
      sc[1] = s;
    } else {
      for (int t = 0; t < T; ++t) { double v = x[t]; if (!is_nan(v)) s += v; }
      sc[2] = s;
    }
  }
  DFM_SYNC();
  if (DFM_TID != 0) return;
  double cnt = sc[0];
  double* lam = Lam ? Lam + (size_t)b * N * r : nullptr;
  bool ok = (mode == 2) ? (cnt > r) : (cnt >= nt_min);
  if (!ok) {
    if (mode != 1 && lam) for (int a = 0; a < r; ++a) lam[i + (size_t)N * a] = DFM_NAN;
    if (mode != 0 && out2) out2[(size_t)b * N + i] = DFM_NAN;
    return;
  }
  double cty[64];                 // copy of rhs (r <= 64 enforced by the host)
  for (int a = 0; a < r; ++a) cty[a] = c[a];
  int bad = chol_solve_packed(A, c, r, 1);
  if (bad) {
    if (st) st[b].status = 3;
    if (mode != 1 && lam) for (int a = 0; a < r; ++a) lam[i + (size_t)N * a] = DFM_NAN;
    if (mode != 0 && out2) out2[(size_t)b * N + i] = DFM_NAN;
    return;
  }
  if (mode == 0 && n_constr > 0) {
    // rows of the stacked constraint that belong to this series
    int nc = 0;
    for (int q = 0; q < n_constr; ++q) if (c_index[q] == i) ++nc;
    if (nc > 0) {
      // tmp = (F'F)^-1 R'  (r x nc), S = R tmp (nc x nc), b -= tmp S^-1 (R b - r_std)
      double* Gp = wk;                       // packed F'F
      double* tmp = Gp + np;                 // r x nc
      double* S = tmp + r * nc;              // packed nc
      double* res = S + nc * (nc + 1) / 2;   // nc
      const double* ftf = FtF + (size_t)b * r * r;
      for (int a = 0; a < r; ++a) for (int cc = 0; cc <= a; ++cc) Gp[pidx(a, cc)] = ftf[a + r * cc];
      int col = 0; bool first = true;
      for (int q = 0; q < n_constr; ++q) {
        if (c_index[q] != i) continue;
        for (int a = 0; a < r; ++a) tmp[a + r * col] = c_R[q + (size_t)n_constr * a];
        if (first) { if (chol_solve_packed(Gp, tmp + r * col, r, 1)) { st[b].status = 3; return; } first = false; }
        else chol_resolve_packed(Gp, tmp + r * col, r, 1);
        double rb = 0.0;
        for (int a = 0; a < r; ++a) rb += c_R[q + (size_t)n_constr * a] * c[a];
        res[col] = rb - c_r[q] / xstd[(size_t)b * N + c_index[q]];   // r_std (:1182-1186)
        ++col;
      }
      int row = 0;
      for (int q = 0; q < n_constr; ++q) {
        if (c_index[q] != i) continue;
        for (int cc = 0; cc <= row; ++cc) {
          double s = 0.0;
          for (int a = 0; a < r; ++a) s += c_R[q + (size_t)n_constr * a] * tmp[a + r * cc];
          S[pidx(row, cc)] = s;
        }
        ++row;
      }
      if (chol_solve_packed(S, res, nc, 1)) { st[b].status = 3; return; }
      for (int a = 0; a < r; ++a) { double s = 0.0; for (int cc = 0; cc < nc; ++cc) s += tmp[a + r * cc] * res[cc]; c[a] -= s; }
    }
  }
  if (mode != 1 && lam) for (int a = 0; a < r; ++a) lam[i + (size_t)N * a] = c[a];
  if (mode != 0 && out2) {
    double bc = 0.0;
    for (int a = 0; a < r; ++a) bc += c[a] * cty[a];
    double ssr = sc[1] - bc;
    if (mode == 1) { double tss = sc[1] - sc[2] * sc[2] / cnt; out2[(size_t)b * N + i] = 1.0 - ssr / tss; }
    else out2[(size_t)b * N + i] = ssr / cnt;
  }
}

// F-step (:364-366): one THREAD per period t; per-thread packed normal equations in shared memory.
// A_t = Lam'Lam - sum_{i missing at t} lam_i lam_i'  (series with NaN Lam are excluded everywhere).
// grid (ceil(T/NT), B); shared: (np + r) * NT + 48 doubles, or 48 when the per-thread systems live in `gsys`
// (global scratch of (np + r) * NT doubles per block, for r whose systems do not fit in shared memory; NULL otherwise).
__global__ void k_als_factor(const double* __restrict__ Xs, const double* __restrict__ LamAll,
                             const double* __restrict__ LtLall, int T, int N, int r, double* __restrict__ Fnew,
                             double* __restrict__ ssr_part, AlsState* st, double* __restrict__ gsys) {
  DFM_SMEM(sm);
  int b = DFM_BY;
  if (st[b].done) return;
  int np = r * (r + 1) / 2;
  int nt = DFM_NT;
  double* sys = gsys ? gsys + ((size_t)b * DFM_GX + DFM_BX) * (np + r) * nt : sm;
  double* A = sys + DFM_TID;                // element e at A[e*nt]
  double* c = sys + (size_t)np * nt + DFM_TID;
  double* red = gsys ? sm : sm + (size_t)(np + r) * nt;
  const double* X = Xs + (size_t)b * T * N;
  const double* Lam = LamAll + (size_t)b * N * r;
  const double* LtL = LtLall + (size_t)b * r * r;
  double* F = Fnew + (size_t)b * T * r;
  double ssr = 0.0;
  for (int t = DFM_BX * nt + DFM_TID; t < T; t += DFM_GX * nt) {
    for (int a = 0; a < r; ++a) { c[a * nt] = 0.0; for (int cc = 0; cc <= a; ++cc) A[pidx(a, cc) * nt] = LtL[a + r * cc]; }
    int nobs = 0;
    for (int i = 0; i < N; ++i) {
      double l0 = Lam[i];
      if (is_nan(l0)) continue;
      double x = X[t + (size_t)T * i];
      if (!is_nan(x)) { ++nobs; for (int a = 0; a < r; ++a) c[a * nt] += x * Lam[i + (size_t)N * a]; }
      else for (int a = 0; a < r; ++a) { double la = Lam[i + (size_t)N * a]; for (int cc = 0; cc <= a; ++cc) A[pidx(a, cc) * nt] -= la * Lam[i + (size_t)N * cc]; }
    }
    int bad = (nobs < r) ? 1 : chol_solve_packed(A, c, r, nt);
    if (bad) { st[b].status = (nobs < r) ? 2 : 3; for (int a = 0; a < r; ++a) c[a * nt] = DFM_NAN; }
    for (int a = 0; a < r; ++a) F[t + (size_t)T * a] = c[a * nt];
    if (!bad)
      for (int i = 0; i < N; ++i) {
        double l0 = Lam[i];
        if (is_nan(l0)) continue;
        double x = X[t + (size_t)T * i];
        if (is_nan(x)) continue;
        double e = x;
        for (int a = 0; a < r; ++a) e -= Lam[i + (size_t)N * a] * c[a * nt];
        ssr += e * e;
      }
  }
  ssr = block_sum(ssr, red);
  if (DFM_TID == 0) ssr_part[(size_t)b * DFM_GX + DFM_BX] = ssr;
}

// SSR total + convergence test (:366-368).  grid (B), 1 thread.
__global__ void k_als_check(AlsState* st, const double* ssr_part, int nblk, double tol, int T, int N,
                            long long max_iter) {
  if (DFM_TID != 0) return;
  int b = DFM_BX;
  if (st[b].done) return;
  double s = 0.0;
  for (int j = 0; j < nblk; ++j) s += ssr_part[(size_t)b * nblk + j];
  st[b].ssr_old = st[b].ssr;
  st[b].ssr = s;
  st[b].iters += 1;
  double diff = fabs(st[b].ssr_old - s);
  if (!(diff >= tol * (double)T * (double)N)) st[b].done = 1;          // `diff >= tol*T*ns || break`
  else if ((long long)st[b].iters >= max_iter) { st[b].done = 1; if (st[b].status == 0) st[b].status = 4; }
  if (st[b].status == 2 || st[b].status == 3) st[b].done = 1;
}

// number of panels not yet done -> *out (device int).  grid (1), 1 block.
__global__ void k_count_active(const AlsState* st, int B, int* out) {
  DFM_SMEM(sm);
  double n = 0.0;
  for (int b = DFM_TID; b < B; b += DFM_NT) n += st[b].done ? 0.0 : 1.0;
  n = block_sum(n, sm);
  if (DFM_TID == 0) *out = (int)n;
}

// ---------------------------------------------------------------- a9 loadings + AR  (:391-415, :295-311)
// One block per series.  data T x ns raw units, F T x r.  Regressors [F 1] (:399), over the rows where y and every factor
// are observed (a missing factor row drops that row for every series, as k_var / k_instability / k_fit_corr do).
// scratch: T doubles per block: y on the usable rows (NaN elsewhere), then the gap-free residual vector.
__global__ void k_loading(const double* __restrict__ dataAll, const double* __restrict__ Fall, int T, int ns, int r,
                          int nt_min, int n_uarlag, double* __restrict__ lambda, double* __restrict__ r2out,
                          double* __restrict__ uar_coef, double* __restrict__ uar_ser, double* __restrict__ scratch,
                          int n_constr, const int* __restrict__ c_index, const double* __restrict__ c_R,
                          const double* __restrict__ c_r, int* __restrict__ status, double* __restrict__ constant,
                          double* __restrict__ resid) {
  DFM_SMEM(sm);
  int s_ = DFM_BX, b = DFM_BY;
  const double* yin = dataAll + ((size_t)b * ns + s_) * T;
  const double* F = Fall + (size_t)b * T * r;
  double* u = scratch + ((size_t)b * ns + s_) * T;
  // drop_missing_row([y F]) (:396): y_t where y_t and every factor are observed, else NaN; the regression reads this copy
  for (int t = DFM_TID; t < T; t += DFM_NT) {
    double v = yin[t];
    for (int a = 0; a < r && !is_nan(v); ++a) if (is_nan(F[t + (size_t)T * a])) v = DFM_NAN;
    u[t] = v;
  }
  DFM_SYNC();
  const double* y = u;
  int K = r + 1, np = K * (K + 1) / 2;
  double* A = sm;               // packed K
  double* c = A + np;           // K
  double* sc = c + K;           // cnt, syy, sy
  double* wk = sc + 4;
  int nwork = np + K + 3;
  for (int e = DFM_TID; e < nwork; e += DFM_NT) {
    double s = 0.0;
    if (e < np) {
      int a = 0; while ((a + 1) * (a + 2) / 2 <= e) ++a;
      int cc = e - a * (a + 1) / 2;
      for (int t = 0; t < T; ++t) if (!is_nan(y[t])) {
        double za = (a < r) ? F[t + (size_t)T * a] : 1.0, zc = (cc < r) ? F[t + (size_t)T * cc] : 1.0;
        s += za * zc;
      }
      A[e] = s;
    } else if (e < np + K) {
      int a = e - np;
      for (int t = 0; t < T; ++t) { double v = y[t]; if (!is_nan(v)) s += v * ((a < r) ? F[t + (size_t)T * a] : 1.0); }
      c[a] = s;
    } else if (e == np + K) { for (int t = 0; t < T; ++t) if (!is_nan(y[t])) s += 1.0; sc[0] = s; }
    else if (e == np + K + 1) { for (int t = 0; t < T; ++t) { double v = y[t]; if (!is_nan(v)) s += v * v; } sc[1] = s; }
    else { for (int t = 0; t < T; ++t) { double v = y[t]; if (!is_nan(v)) s += v; } sc[2] = s; }
  }
  DFM_SYNC();
  if (DFM_TID != 0) return;
  size_t o = (size_t)b * ns + s_;
  double* lam = lambda + (size_t)b * ns * r;
  double* ac = uar_coef + (size_t)b * ns * n_uarlag;
  int cnt = (int)sc[0];
  // every early exit leaves NaN in ALL outputs of this series (never stale workspace contents)
#define LOAD_NAN_ALL() do {                                                                       \
    for (int a = 0; a < r; ++a) lam[s_ + (size_t)ns * a] = DFM_NAN;                               \
    r2out[o] = DFM_NAN; uar_ser[o] = DFM_NAN;                                                     \
    for (int l = 0; l < n_uarlag; ++l) ac[s_ + (size_t)ns * l] = DFM_NAN;                         \
    if (constant) constant[o] = DFM_NAN;                                                          \
    if (resid) for (int t = 0; t < T; ++t) resid[o * T + t] = DFM_NAN;                            \
  } while (0)
  if (cnt < nt_min) {            // reference leaves these undefined (SURVEY 'bugs'): NaN
    LOAD_NAN_ALL();
    return;
  }
  bool constrained = false;
  for (int q = 0; q < n_constr; ++q) if (c_index[q] == s_) constrained = true;
  if (chol_solve_packed(A, c, K, 1)) { status[b] = 3; LOAD_NAN_ALL(); return; }
  if (constrained) {             // :loading constraint: R_tmp = [R 0], r unstandardized (:1147-1148)
    int nc = 0;
    for (int q = 0; q < n_constr; ++q) if (c_index[q] == s_) ++nc;
    double* tmp = wk;            // K x nc
    double* S = tmp + K * nc;
    double* res = S + nc * (nc + 1) / 2;
    int col = 0;
    for (int q = 0; q < n_constr; ++q) {
      if (c_index[q] != s_) continue;
      for (int a = 0; a < r; ++a) tmp[a + K * col] = c_R[q + (size_t)n_constr * a];
      tmp[r + K * col] = 0.0;
      chol_resolve_packed(A, tmp + K * col, K, 1);
      double rb = 0.0;
      for (int a = 0; a < r; ++a) rb += c_R[q + (size_t)n_constr * a] * c[a];
      res[col] = rb - c_r[q];
      ++col;
    }
    int row = 0;
    for (int q = 0; q < n_constr; ++q) {
      if (c_index[q] != s_) continue;
      for (int cc = 0; cc <= row; ++cc) {
        double s = 0.0;
        for (int a = 0; a < r; ++a) s += c_R[q + (size_t)n_constr * a] * tmp[a + K * cc];
        S[pidx(row, cc)] = s;
      }
      ++row;
    }
    if (chol_solve_packed(S, res, nc, 1)) { status[b] = 3; LOAD_NAN_ALL(); return; }
    for (int a = 0; a < K; ++a) { double s = 0.0; for (int cc = 0; cc < nc; ++cc) s += tmp[a + K * cc] * res[cc]; c[a] -= s; }
  }
  for (int a = 0; a < r; ++a) lam[s_ + (size_t)ns * a] = c[a];
  if (constant) constant[o] = c[r];
  // gap-free residuals (:400), R2 (:404 via compute_r2 :565-569)
  int n = 0; double ssr = 0.0;
  for (int t = 0; t < T; ++t) {
    double v = y[t];
    if (is_nan(v)) { if (resid) resid[o * T + t] = DFM_NAN; continue; }
    double e = v - c[r];
    for (int a = 0; a < r; ++a) e -= c[a] * F[t + (size_t)T * a];
    if (resid) resid[o * T + t] = e;
    u[n++] = e; ssr += e * e;
  }
  double tss = sc[1] - sc[2] * sc[2] / cnt;
  double R2 = 1.0 - ssr / tss;
  r2out[o] = R2;
  if (!(R2 < 0.9999)) {          // :405-409
    for (int l = 0; l < n_uarlag; ++l) ac[s_ + (size_t)ns * l] = 0.0;
    uar_ser[o] = 0.0;
    return;
  }
  // uar (:305-311): regress u[j] on u[j-1..j-L], j = L..n-1; ser = sqrt(ssr/(n - L))
  int L = n_uarlag, npl = L * (L + 1) / 2;
  double* AA = wk; double* cc2 = AA + npl;
  for (int e = 0; e < npl + L; ++e) AA[e] = 0.0;
  for (int j = L; j < n; ++j)
    for (int a = 0; a < L; ++a) {
      double ua = u[j - 1 - a];
      cc2[a] += ua * u[j];
      for (int q = 0; q <= a; ++q) AA[pidx(a, q)] += ua * u[j - 1 - q];
    }
  if (n - L < L || chol_solve_packed(AA, cc2, L, 1)) {
    status[b] = 3; uar_ser[o] = DFM_NAN;
    for (int l = 0; l < L; ++l) ac[s_ + (size_t)ns * l] = DFM_NAN;
    return;
  }
  double ssr2 = 0.0;
  for (int j = L; j < n; ++j) { double e = u[j]; for (int a = 0; a < L; ++a) e -= cc2[a] * u[j - 1 - a]; ssr2 += e * e; }
  for (int l = 0; l < L; ++l) ac[s_ + (size_t)ns * l] = cc2[l];
  uar_ser[o] = sqrt(ssr2 / (double)(n - L));
#undef LOAD_NAN_ALL
}

// ---------------------------------------------------------------- a10 factor VAR (:444-492)
// grid (B), one block.  Regressors [1, y_{t-1}, ..., y_{t-p}] (const first, :451).  dof_mode 0:
// seps = e'e/(T_used - K) (:460-461); dof_mode 1: e'e/T_used (EM initialisation).
// shared: K*K + K*r + 64 doubles.
__global__ void k_var(const double* __restrict__ Fall, int T, int r, int p, int withconst, int dof_mode,
                      double* __restrict__ betahat, double* __restrict__ resid, double* __restrict__ seps,
                      double* __restrict__ Mo, double* __restrict__ Qo, double* __restrict__ Go, double* __restrict__ Ao,
                      int* __restrict__ status) {
  DFM_SMEM(sm);
  int b = DFM_BX;
  const double* F = Fall + (size_t)b * T * r;
  int k = r * p, K = k + (withconst ? 1 : 0), Tu = T - p;
  double* ZZ = sm;                 // K x K
  double* ZY = ZZ + K * K;         // K x r  -> beta
  double* Se = ZY + K * r;         // r x r
  int* info = (int*)(Se + r * r);       // [0] = Cholesky flag, [1] = number of rows kept
  unsigned char* keep = (unsigned char*)(info + 4);      // [T]: row t enters the regression
  if (DFM_TID == 0) { info[0] = 0; info[1] = 0; }
  DFM_SYNC();
  // estimate_var! regresses with ols_skipmissing(..., Balanced()) (dfm_functions.ipynb:242-252, 452): every row with a
  // missing y_t or a missing lag is dropped; rows t < p have no lags and are always dropped
  {
    int cnt = 0;
    for (int t = DFM_TID; t < T; t += DFM_NT) {
      bool ok = t >= p;
      for (int l = 0; ok && l <= p; ++l) for (int c = 0; c < r; ++c) if (is_nan(F[(t - l) + (size_t)T * c])) { ok = false; break; }
      keep[t] = ok ? 1 : 0; cnt += ok ? 1 : 0;
    }
    if (cnt) atomicAdd(&info[1], cnt);
  }
  DFM_SYNC();
  Tu = info[1];
  // a failed panel leaves NaN in every output (so that a batched caller can drop it) and its code in status[b]
#define VAR_FAIL(code_) do {                                                                                        \
    if (DFM_TID == 0) status[b] = (code_);                                                                          \
    for (int e = DFM_TID; e < T * r; e += DFM_NT) resid[(size_t)b * T * r + e] = DFM_NAN;                           \
    if (betahat) for (int e = DFM_TID; e < K * r; e += DFM_NT) betahat[(size_t)b * K * r + e] = DFM_NAN;            \
    if (seps) for (int e = DFM_TID; e < r * r; e += DFM_NT) seps[(size_t)b * r * r + e] = DFM_NAN;                  \
    if (Mo) for (int e = DFM_TID; e < k * k; e += DFM_NT) Mo[(size_t)b * k * k + e] = DFM_NAN;                      \
    if (Ao) for (int e = DFM_TID; e < r * k; e += DFM_NT) Ao[(size_t)b * r * k + e] = DFM_NAN;                      \
    if (Qo) for (int e = DFM_TID; e < r * k; e += DFM_NT) Qo[(size_t)b * r * k + e] = DFM_NAN;                      \
    if (Go) for (int e = DFM_TID; e < k * r; e += DFM_NT) Go[(size_t)b * k * r + e] = DFM_NAN;                      \
    return;                                                                                                         \
  } while (0)
  if (Tu <= K) VAR_FAIL(2);
  // regressor j at time t (t = p..T-1): j==0&&const -> 1 ; else lag l = (j-c)/r + 1, var = (j-c)%r
#define ZREG(t, j) ((withconst && (j) == 0) ? 1.0 : F[((t) - (((j) - (withconst ? 1 : 0)) / r + 1)) + (size_t)T * (((j) - (withconst ? 1 : 0)) % r)])
  for (int e = DFM_TID; e < K * K; e += DFM_NT) {
    int a = e % K, c = e / K;
    if (a < c) continue;
    double s = 0.0;
    for (int t = p; t < T; ++t) if (keep[t]) s += ZREG(t, a) * ZREG(t, c);
    ZZ[a + K * c] = s; ZZ[c + K * a] = s;
  }
  for (int e = DFM_TID; e < K * r; e += DFM_NT) {
    int a = e % K, c = e / K;
    double s = 0.0;
    for (int t = p; t < T; ++t) if (keep[t]) s += ZREG(t, a) * F[t + (size_t)T * c];
    ZY[a + K * c] = s;
  }
  DFM_SYNC();
  bm_chol(ZZ, K, K, info);
  bm_trsm_lower(ZZ, K, K, ZY, K, r);
  bm_trsm_lowerT(ZZ, K, K, ZY, K, r);          // ZY = betahat (K x r)
  double* res = resid + (size_t)b * T * r;
  if (*info) VAR_FAIL(3);
  // residuals -> global (needed for seps); dropped rows are NaN (:464 writes the kept rows only)
  for (int e = DFM_TID; e < T * r; e += DFM_NT) {
    int t = e % T, c = e / T;
    double v = DFM_NAN;
    if (keep[t]) { v = F[t + (size_t)T * c]; for (int a = 0; a < K; ++a) v -= ZREG(t, a) * ZY[a + K * c]; }
    res[t + (size_t)T * c] = v;
  }
  DFM_SYNC();
#undef ZREG
  double ndf = dof_mode ? (double)Tu : (double)(Tu - K);
  for (int e = DFM_TID; e < r * r; e += DFM_NT) {
    int a = e % r, c = e / r;
    double s = 0.0;
    for (int t = p; t < T; ++t) if (keep[t]) s += res[t + (size_t)T * a] * res[t + (size_t)T * c];
    Se[a + r * c] = s / ndf;
  }
  DFM_SYNC();
  if (betahat) for (int e = DFM_TID; e < K * r; e += DFM_NT) betahat[(size_t)b * K * r + e] = ZY[e];
  if (seps) for (int e = DFM_TID; e < r * r; e += DFM_NT) seps[(size_t)b * r * r + e] = Se[e];
  // companion matrices (:477-492)
  int c0 = withconst ? 1 : 0;
  if (Mo) for (int e = DFM_TID; e < k * k; e += DFM_NT) {
    int i = e % k, j = e / k;
    double v = 0.0;
    if (i < r) v = ZY[(c0 + j) + K * i];            // b = betahat[2:end,:]'
    else if (j == i - r) v = 1.0;
    Mo[(size_t)b * k * k + e] = v;
  }
  if (Ao) for (int e = DFM_TID; e < r * k; e += DFM_NT) { int i = e % r, j = e / r; Ao[(size_t)b * r * k + e] = ZY[(c0 + j) + K * i]; }
  if (Qo) for (int e = DFM_TID; e < r * k; e += DFM_NT) { int i = e % r, j = e / r; Qo[(size_t)b * r * k + e] = (i == j) ? 1.0 : 0.0; }
  DFM_SYNC();
  if (Go) {
    bm_chol(Se, r, r, info);                           // lower factor = cholesky(seps).U'
    if (*info) VAR_FAIL(3);
    for (int e = DFM_TID; e < k * r; e += DFM_NT) { int i = e % k, j = e / k; Go[(size_t)b * k * r + e] = (i < r) ? Se[i + r * j] : 0.0; }
  }
#undef VAR_FAIL
}

// ---------------------------------------------------------------- a11 IRF (:793-816)
// grid (n_shock, B), one block per shock; shared irf_smem_doubles(k) (x and x2, 2k doubles, and 8 spare).
__host__ __device__ inline size_t irf_smem_doubles(int k) { return 2 * (size_t)k + 8; }

__global__ void k_irf(const double* __restrict__ Mall, const double* __restrict__ Qall, const double* __restrict__ Gall,
                      int k, int r, int H, int n_shock, const int* __restrict__ shock_ids, double* __restrict__ irf) {
  DFM_SMEM(sm);
  int j = DFM_BX, b = DFM_BY;
  const double* M = Mall + (size_t)b * k * k; const double* Q = Qall + (size_t)b * r * k;
  const double* G = Gall + (size_t)b * k * r;
  double* x = sm; double* x2 = sm + k;
  double* out = irf + ((size_t)b * n_shock + j) * r * H;
  for (int i = DFM_TID; i < k; i += DFM_NT) x[i] = G[i + (size_t)k * shock_ids[j]];
  DFM_SYNC();
  for (int h = 0; h < H; ++h) {
    for (int i = DFM_TID; i < r; i += DFM_NT) { double s = 0.0; for (int l = 0; l < k; ++l) s += Q[i + (size_t)r * l] * x[l]; out[i + (size_t)r * h] = s; }
    for (int i = DFM_TID; i < k; i += DFM_NT) { double s = 0.0; for (int l = 0; l < k; ++l) s += M[i + (size_t)k * l] * x[l]; x2[i] = s; }
    DFM_SYNC();
    for (int i = DFM_TID; i < k; i += DFM_NT) x[i] = x2[i];
    DFM_SYNC();
  }
}

}  // namespace dfm
