// dfm_kernels_news.cuh -- the news decomposition of a nowcast revision (dfm_news): the revision of a target
// y = x_{i*, t*} between two data vintages, E[y | new] - E[y | old] = sum_j w_j I_j, as a sum over the newly released cells
// j of their news I_j = x_j - E[x_j | old] times the weights w = Cov(y, I | old) Var(I | old)^-1 (Banbura & Modugno 2014),
// at fixed state-space parameters.  The spec is tests/news_oracle.py.  After the fixed-parameter E-step of
// dfm_kalman_smooth on the OLD vintage (same kernels, same scratch) four kernels run:
//   k_news_window   one CTA per pair: the news mask of the release window (X_old NaN, X_new observed, series in the model),
//                   the consistency of the two vintages (status DFM_ERR_ARG), and the sorted set P of the periods that
//                   hold a news cell or a target (W of them)
//   k_news_cov      one CTA per pair: the RTS covariance recursion backwards from the last period to min P with the
//                   smoother gains J_t = P_{t|t} M' P_{t+1|t}^-1, the joint covariance Sigma of (f_s)_{s in P}
//                   (Cov(z_s, z_t) = J_s .. J_{t-1} Ps_t), L = PSD Cholesky factor of Sigma, S = I + L' C^J L with
//                   C^J = blockdiag(sum_{j news at s} lam_j lam_j' / R_j), and g_q = L S^-1 L' (e_{t*} x lam_{i*}) -- the
//                   Woodbury form of Cov(y, I) Var(I)^-1 without an n_news x n_news matrix; every k x k and W r x W r
//                   product is a DMMA tile product (wt_gemm); old_est of each target
//   k_news_project  tiles of window rows x series: E[x | old] = F_old Lam' and w = [g] Lam' o (1 / R) as DMMA tile products,
//                   I = X_new - E[x | old] at the news cells, coalesced writes of the requested outputs, and the partial
//                   sums of the contributions w I per (tile, target)
//   k_news_finish   new_est = old_est + the partial sums of the tiles in a fixed order (bit-reproducible run to run)
#pragma once
#include "dfm_common.cuh"
#include "dfm_kernels_em.cuh"
#include "dfm_kernels_ss.cuh"
#include "dfm_kernels_sim.cuh"

namespace dfm {

#define NEWS_MAXN 128          // W r: the factors of the periods that matter
#define NEWS_MAXQ 64           // targets per call
#define NEWS_TP 8              // window rows per tile of k_news_project
#define NEWS_NS 64             // series per tile of k_news_project
#define NEWS_QC 8              // targets per DMMA pass of k_news_project

// How a target's revision is formed (per pair and target)
enum { NEWS_MODEL = 0,         // by the weights g_q' lam_i / R_i
       NEWS_OBSERVED = 1,      // observed in the old vintage: revision 0, weights 0
       NEWS_RELEASED = 2,      // a news cell itself: weight 1 on its own cell, 0 elsewhere
       NEWS_OUT = 3 };         // series out of the model: NaN

__host__ __device__ inline size_t news_window_smem_bytes(int nr, int nq) { return (size_t)(2 * nr + nq + 2) * sizeof(int); }

// Per pair b: mask [nr x N] (window row t, series i at t + nr i) = 1 at a news cell; plist [Wmax + 1] = W, then the sorted
// periods of P; rowp [nr] = the index in P of window row t, or -1; pstat = DFM_ERR_ARG if the vintages are inconsistent (a
// cell of X_old missing or changed in X_new, or a new cell above the window -- checked here when Xabove is given, by the
// caller otherwise, who then sets pstat to 1 before the launch), else the E-step's status.  Xo: the padded old panels
// [Tp x N]; the window rows of X_new at Xn[(b N + i) ldn + row0 + t]; Xabove: X_new [T x N] in full, or NULL.
// grid (B), 256 threads.
__global__ void k_news_window(const double* __restrict__ Xo_, const double* __restrict__ Xn, int ldn, int row0,
                              const double* __restrict__ Xabove, const double* __restrict__ LamAll, const double* __restrict__ Rall,
                              const int* __restrict__ tper, int nq, const int* __restrict__ estat, int T, int Tp, int N, int r,
                              int nr, int Wmax, unsigned char* __restrict__ mask_, int* __restrict__ plist_, int* __restrict__ rowp_,
                              int* __restrict__ pstat) {
  DFM_SMEM(sm);
  int* rowf = (int*)sm;                                // [nr]       does window row t hold a news cell?
  int* cand = rowf + nr;                               // [nr + nq]  candidate periods of P
  int* bad = cand + nr + nq;
  const int b = DFM_BX, w0 = T - nr;
  const double* Xo = Xo_ + (size_t)b * Tp * N;
  const double* Lam = LamAll + (size_t)b * N * r;
  const double* R = Rall + (size_t)b * N;
  unsigned char* mask = mask_ + (size_t)b * nr * N;
  for (int t = DFM_TID; t < nr; t += DFM_NT) rowf[t] = 0;
  if (DFM_TID == 0) *bad = pstat[b];
  DFM_SYNC();
  for (long long e = DFM_TID; e < (long long)nr * N; e += DFM_NT) {
    const int i = (int)(e / nr), t = (int)(e - (long long)i * nr);
    const double x0 = Xo[(size_t)i * Tp + w0 + t], x1 = Xn[((size_t)b * N + i) * ldn + row0 + t];
    unsigned char m = 0;
    if (!is_nan(x0)) { if (is_nan(x1) || x1 != x0) *bad = 1; }          // (benign race: all store 1)
    else if (!is_nan(x1) && !is_nan(Lam[i]) && !is_nan(R[i])) { m = 1; rowf[t] = 1; }
    mask[e] = m;
  }
  if (Xabove && w0 > 0)
    for (long long e = DFM_TID; e < (long long)w0 * N; e += DFM_NT) {
      const int i = (int)(e / w0), t = (int)(e - (long long)i * w0);
      const double x0 = Xo[(size_t)i * Tp + t], x1 = Xabove[((size_t)b * N + i) * T + t];
      if (is_nan(x0) != is_nan(x1) || (!is_nan(x0) && x0 != x1)) *bad = 1;
    }
  DFM_SYNC();
  if (DFM_TID == 0) {
    int nc = 0;
    for (int t = 0; t < nr; ++t) if (rowf[t]) cand[nc++] = w0 + t;
    for (int q = 0; q < nq; ++q) cand[nc++] = tper[q];
    for (int a = 1; a < nc; ++a) {                     // insertion sort (nc <= nr + nq)
      const int v = cand[a];
      int c = a - 1;
      while (c >= 0 && cand[c] > v) { cand[c + 1] = cand[c]; --c; }
      cand[c + 1] = v;
    }
    int W = 0;
    int* plist = plist_ + (size_t)b * (Wmax + 1);
    for (int a = 0; a < nc; ++a) if (W == 0 || cand[a] != plist[W]) plist[1 + W++] = cand[a];
    plist[0] = W;
    for (int t = 0; t < nr; ++t) {
      int ix = -1;
      for (int a = 0; a < W; ++a) if (plist[1 + a] == w0 + t) ix = a;
      rowp_[(size_t)b * nr + t] = ix;
    }
    pstat[b] = *bad ? 1 : estat[b];
  }
}

// Shared memory of k_news_cov: the k x k part always; the W r-sized part (Xc double buffer k x nmax, Sigma -> L and S
// nmax x nmax, U nmax x nq, C_a L_a r x nmax) too when it fits, else it lives in global scratch (news_cov_big_doubles per
// pair).
__host__ __device__ inline size_t news_cov_small_doubles(int r, int p) {
  const size_t k = (size_t)r * p;
  return 7 * k * k + 8 + NEWS_MAXQ;
}
__host__ __device__ inline size_t news_cov_big_doubles(int r, int p, int nmax, int nq) {
  const size_t k = (size_t)r * p, n = (size_t)nmax;
  return 2 * k * n + 2 * n * n + n * nq + (size_t)r * n;
}

// One CTA per pair.  A [r x k], the E-step's P_{t+1|t} (Ppg) and P_{t|t} (Pfg) at the explicit periods with src[t] (the
// period whose covariances period t uses), Fs [Tp x r] = E[f_t | old], Xo the padded old panel [Tp x N].  Outputs per pair:
// gv [nq][nmax] = g_q (block a of P at a r), kind [nq], oldv [nq] = E[y_q | old].  big_g: global scratch of the W r-sized
// part, or NULL when it is in shared memory.  Pairs with pstat != 0 are skipped (k_news_finish writes their NaN).
__global__ void k_news_cov(const double* __restrict__ Aall, const double* __restrict__ Ppg_, const double* __restrict__ Pfg_,
                           const int* __restrict__ src_, const double* __restrict__ Fs_, const double* __restrict__ Xo_,
                           const double* __restrict__ LamAll, const double* __restrict__ Rall, const unsigned char* __restrict__ mask_,
                           const int* __restrict__ plist_, const int* __restrict__ tser, const int* __restrict__ tper, int nq,
                           const int* __restrict__ pstat, int T, int Tp, int N, int r, int p, int nr, int Wmax,
                           double* __restrict__ big_g, double* __restrict__ gv_, int* __restrict__ kind_, double* __restrict__ oldv_) {
  DFM_SMEM(sm);
  const int b = DFM_BX, k = r * p, kk = k * k, nmax = Wmax * r, w0 = T - nr;
  if (pstat[b] != 0) return;
  const double* A = Aall + (size_t)b * r * k;
  const double* Ppg = Ppg_ + (size_t)b * Tp * kk;
  const double* Pfg = Pfg_ + (size_t)b * Tp * kk;
  const int* src = src_ + (size_t)b * Tp;
  const double* Fs = Fs_ + (size_t)b * Tp * r;
  const double* Xo = Xo_ + (size_t)b * Tp * N;
  const double* Lam = LamAll + (size_t)b * N * r;
  const double* R = Rall + (size_t)b * N;
  const unsigned char* mask = mask_ + (size_t)b * nr * N;
  const int* plist = plist_ + (size_t)b * (Wmax + 1);
  const int W = plist[0], n = W * r;
  const int* P = plist + 1;
  double* M = sm;      double* Pf = M + kk;   double* Pp = Pf + kk;  double* Ps = Pp + kk;
  double* J = Ps + kk; double* T1 = J + kk;   double* T2 = T1 + kk;
  int* info = (int*)(T2 + kk);                         // [0] Cholesky flag, [8 ..] kind, [8 + NEWS_MAXQ ..] P index of the targets
  int* kindS = info + 8;
  int* aqS = kindS + NEWS_MAXQ;
  double* big = big_g ? big_g + (size_t)b * news_cov_big_doubles(r, p, nmax, nq) : sm + news_cov_small_doubles(r, p);
  double* Xc[2] = {big, big + (size_t)k * nmax};       // [k x nmax]   Cov(z_t, f_{s_b}) of the periods s_b > t of P
  double* Sg = big + 2 * (size_t)k * nmax;             // [n x n]      Sigma, then L
  double* S = Sg + (size_t)nmax * nmax;                // [n x n]      S = I + L' C^J L, then its Cholesky factor
  double* U = S + (size_t)nmax * nmax;                 // [n x nq]     L' (e_{t*} x lam_{i*}), then S^-1 of it
  double* Tb = U + (size_t)nmax * nq;                  // [r x n]      C_a L_a
  for (int e = DFM_TID; e < kk; e += DFM_NT) {
    const int i = e % k, j = e / k;
    M[e] = (i < r) ? A[i + r * j] : ((j == i - r) ? 1.0 : 0.0);
  }
  if (DFM_TID == 0) info[0] = 0;
  DFM_SYNC();
  // ---- backwards from the last period: Ps_t, J_t, and the blocks of Sigma at the periods of P
  int a = W - 1, cur = 0, js0 = -1, js1 = -1;
  for (int t = Tp - 1; t >= P[0]; --t) {
    if (t == Tp - 1) {
      for (int e = DFM_TID; e < kk; e += DFM_NT) Ps[e] = Pfg[(size_t)src[t] * kk + e];
      DFM_SYNC();
    } else {
      const int sf = src[t], sp = src[t + 1];
      for (int e = DFM_TID; e < kk; e += DFM_NT) T2[e] = Ps[e] - Ppg[(size_t)sp * kk + e];      // D = Ps_{t+1} - P_{t+1|t}
      if (sf != js0 || sp != js1) {                    // a frozen period's gain is its source periods' gain
        for (int e = DFM_TID; e < kk; e += DFM_NT) { Pf[e] = Pfg[(size_t)sf * kk + e]; Pp[e] = Ppg[(size_t)sp * kk + e]; }
        DFM_SYNC();
        wt_gemm(M, 1, k, Pf, k, 1, k, k, k, [&](int i, int j, double v) { T1[i + k * j] = v; });     // M Pf
        DFM_SYNC();
        bm_chol(Pp, k, k, info);
        bm_trsm_lower(Pp, k, k, T1, k, k);
        bm_trsm_lowerT(Pp, k, k, T1, k, k);                                                       // Pp^-1 M Pf = J'
        for (int e = DFM_TID; e < kk; e += DFM_NT) { const int i = e % k, j = e / k; J[e] = T1[j + k * i]; }
        js0 = sf; js1 = sp;
      }
      DFM_SYNC();
      wt_gemm(J, 1, k, T2, k, 1, k, k, k, [&](int i, int j, double v) { T1[i + k * j] = v; });        // J D
      DFM_SYNC();
      wt_gemm(T1, 1, k, J, 1, k, k, k, k, [&](int i, int j, double v) { Ps[i + k * j] = Pf[i + k * j] + v; });   // Pf + J D J'
      const int c0 = (a + 1) * r;
      if (c0 < n) {                                    // Cov(z_t, f_{s_b}) = J_t Cov(z_{t+1}, f_{s_b})
        double* Xn = Xc[cur ^ 1];
        wt_gemm(J, 1, k, Xc[cur] + (size_t)k * c0, k, 1, k, n - c0, k, [&](int i, int j, double v) { Xn[i + (size_t)k * (c0 + j)] = v; });
        cur ^= 1;
      }
      DFM_SYNC();
    }
    if (a >= 0 && t == P[a]) {
      const int c0 = a * r, nb = n - c0 - r;
      const double* X = Xc[cur];
      for (int e = DFM_TID; e < r * r; e += DFM_NT) { const int c = e % r, d = e / r; Sg[c0 + c + (size_t)n * (c0 + d)] = Ps[c + k * d]; }
      for (int e = DFM_TID; e < nb * r; e += DFM_NT) {                 // blocks below: Cov(f_{s_b}, f_{s_a}), b > a
        const int m = c0 + r + e % nb, d = e / nb;
        Sg[m + (size_t)n * (c0 + d)] = X[d + (size_t)k * m];
      }
      double* Xw = Xc[cur];
      for (int e = DFM_TID; e < k * r; e += DFM_NT) { const int i = e % k, d = e / k; Xw[i + (size_t)k * (c0 + d)] = Ps[i + k * d]; }
      --a;
      DFM_SYNC();
    }
  }
  // ---- L, S = I + L' C^J L (block by block of P), its Cholesky factor
  for (int e = DFM_TID; e < n * n; e += DFM_NT) S[e] = (e % n == e / n) ? 1.0 : 0.0;
  DFM_SYNC();
  bm_chol_psd(Sg, n, n);
  for (int b2 = 0; b2 < W; ++b2) {
    const int s = P[b2];
    if (s < w0 || s >= T) continue;
    const int tw = s - w0;
    for (int e = DFM_TID; e < r * r; e += DFM_NT) {    // C_a = sum over the news cells of the row (series order)
      const int c = e % r, d = e / r;
      double v = 0.0;
      for (int i = 0; i < N; ++i)
        if (mask[tw + (size_t)nr * i]) v += Lam[i + (size_t)N * c] * Lam[i + (size_t)N * d] / R[i];
      T2[e] = v;
    }
    DFM_SYNC();
    wt_gemm(T2, 1, r, Sg + b2 * r, n, 1, r, n, r, [&](int c, int j, double v) { Tb[c + (size_t)r * j] = v; });         // C_a L_a
    DFM_SYNC();
    wt_gemm(Sg + b2 * r, n, 1, Tb, r, 1, n, n, r, [&](int m, int j, double v) { S[m + (size_t)n * j] += v; });       // += L_a' C_a L_a
    DFM_SYNC();
  }
  bm_chol(S, n, n, info);
  // ---- the targets: kind, old_est, and U = L' (e_{t*} x lam_{i*}) for those the weights carry
  for (int q = DFM_TID; q < nq; q += DFM_NT) {
    const int i = tser[q], t = tper[q];
    int kd; double o;
    if (is_nan(Lam[i]) || is_nan(R[i])) { kd = NEWS_OUT; o = DFM_NAN; }
    else {
      double f = 0.0;
      for (int c = 0; c < r; ++c) f += Lam[i + (size_t)N * c] * Fs[t + (size_t)Tp * c];
      const double x = (t < T) ? Xo[(size_t)i * Tp + t] : DFM_NAN;
      if (!is_nan(x)) { kd = NEWS_OBSERVED; o = x; }
      else if (t >= w0 && t < T && mask[(t - w0) + (size_t)nr * i]) { kd = NEWS_RELEASED; o = f; }
      else { kd = NEWS_MODEL; o = f; }
    }
    int aq = 0;
    for (int c = 0; c < W; ++c) if (P[c] == t) aq = c;
    kindS[q] = kd; aqS[q] = aq;
    kind_[(size_t)b * nq + q] = kd; oldv_[(size_t)b * nq + q] = o;
  }
  DFM_SYNC();
  for (int e = DFM_TID; e < n * nq; e += DFM_NT) {
    const int m = e % n, q = e / n, i = tser[q];
    double v = 0.0;
    if (kindS[q] == NEWS_MODEL)
      for (int c = 0; c < r; ++c) v += Sg[aqS[q] * r + c + (size_t)n * m] * Lam[i + (size_t)N * c];
    U[m + (size_t)n * q] = v;
  }
  DFM_SYNC();
  bm_trsm_lower(S, n, n, U, n, nq);
  bm_trsm_lowerT(S, n, n, U, n, nq);
  double* gv = gv_ + (size_t)b * nq * nmax;
  wt_gemm(Sg, 1, n, U, n, 1, n, nq, n, [&](int m, int q, double v) { gv[(size_t)q * nmax + m] = v; });                // g = L S^-1 U
}

__host__ __device__ inline size_t news_project_smem_doubles(int r) {
  const size_t ld = (size_t)em_lds(r);
  return (size_t)NEWS_NS * ld + (size_t)NEWS_TP * ld + (size_t)NEWS_QC * NEWS_TP * ld + (size_t)NEWS_NS * (NEWS_TP + 1) +
         (size_t)NEWS_NS * (NEWS_QC * NEWS_TP + 1) + NEWS_NS + 40 + (NEWS_NS * NEWS_TP + NEWS_TP + 1) / 2 + 1;
}

// Tile of NEWS_TP window rows x NEWS_NS series of one pair: news [nr x N], weight / contrib [nr x N x nq] (may be NULL), and
// part [ntile x nq] the tile's sum of the contributions of each target (sum over the tile's threads in a fixed order).
// Fs, Lam, R as k_news_cov; the window rows of X_new as in k_news_window.  grid (ceil(nr / NEWS_TP), ceil(N / NEWS_NS) * nb),
// 256 threads; pairs b0 .. b0 + nb - 1.
__global__ void k_news_project(const double* __restrict__ Fs_, const double* __restrict__ Xn, int ldn, int row0,
                               const double* __restrict__ LamAll, const double* __restrict__ Rall, const unsigned char* __restrict__ mask_,
                               const int* __restrict__ rowp_, const double* __restrict__ gv_, const int* __restrict__ kind_,
                               const int* __restrict__ tser, const int* __restrict__ tper, int nq, const int* __restrict__ pstat,
                               int T, int Tp, int N, int r, int nr, int Wmax, int b0, double* __restrict__ news,
                               double* __restrict__ weight, double* __restrict__ contrib, double* __restrict__ part) {
  DFM_SMEM(sm);
  const int nst = (N + NEWS_NS - 1) / NEWS_NS;
  const int b = b0 + DFM_BY / nst, i0 = (DFM_BY % nst) * NEWS_NS, t0 = DFM_BX * NEWS_TP;
  const int ni = (N - i0 < NEWS_NS) ? N - i0 : NEWS_NS, nt = (nr - t0 < NEWS_TP) ? nr - t0 : NEWS_TP;
  const int ld = em_lds(r), ldc = NEWS_TP + 1, MQ = NEWS_QC * NEWS_TP, ldw = MQ + 1, nmax = Wmax * r, w0 = T - nr;
  const int ntile = DFM_GX * nst, tile = DFM_BX * nst + DFM_BY % nst;
  const size_t onr = (size_t)nr * N;
  double* Ls = sm;                                     // [NEWS_NS][ld]   loadings of the tile's series
  double* Fsh = Ls + (size_t)NEWS_NS * ld;             // [NEWS_TP][ld]   E[f_t | old] of the tile's rows
  double* Gs = Fsh + (size_t)NEWS_TP * ld;             // [MQ][ld]        g_{q, s(t)} of NEWS_QC targets
  double* Is = Gs + (size_t)MQ * ld;                   // [NEWS_NS][ldc]  E[x | old], then the news
  double* Wt = Is + (size_t)NEWS_NS * ldc;             // [NEWS_NS][ldw]  g' lam_i of (target, row)
  double* Rs = Wt + (size_t)NEWS_NS * ldw;             // [NEWS_NS]
  double* red = Rs + NEWS_NS;                          // [40]
  int* Ms = (int*)(red + 40);                          // [NEWS_NS][NEWS_TP]  news mask
  int* Rp = Ms + NEWS_NS * NEWS_TP;                    // [NEWS_TP]           P index of the row, or -1
  if (pstat[b] != 0) {
    for (int e = DFM_TID; e < ni * NEWS_TP; e += DFM_NT) {
      const int i = e / NEWS_TP, t = e - i * NEWS_TP;
      if (t >= nt) continue;
      const size_t g = (size_t)(i0 + i) * nr + t0 + t;
      if (news) news[(size_t)b * onr + g] = DFM_NAN;
      for (int q = 0; q < nq; ++q) {
        if (weight) weight[((size_t)b * nq + q) * onr + g] = DFM_NAN;
        if (contrib) contrib[((size_t)b * nq + q) * onr + g] = DFM_NAN;
      }
    }
    for (int q = DFM_TID; q < nq; q += DFM_NT) part[((size_t)b * ntile + tile) * nq + q] = DFM_NAN;
    return;
  }
  const double* Lam = LamAll + (size_t)b * N * r;
  const double* R = Rall + (size_t)b * N;
  const double* Fs = Fs_ + (size_t)b * Tp * r;
  const unsigned char* mask = mask_ + (size_t)b * onr;
  const double* gv = gv_ + (size_t)b * nq * nmax;
  for (int e = DFM_TID; e < NEWS_NS * r; e += DFM_NT) {
    const int i = e % NEWS_NS, c = e / NEWS_NS;
    Ls[i * ld + c] = (i < ni) ? Lam[i0 + i + (size_t)N * c] : 0.0;
  }
  for (int i = DFM_TID; i < NEWS_NS; i += DFM_NT) Rs[i] = (i < ni) ? R[i0 + i] : 1.0;
  for (int e = DFM_TID; e < NEWS_TP * r; e += DFM_NT) {
    const int t = e % NEWS_TP, c = e / NEWS_TP;
    Fsh[t * ld + c] = (t < nt) ? Fs[w0 + t0 + t + (size_t)Tp * c] : 0.0;
  }
  for (int e = DFM_TID; e < NEWS_NS * NEWS_TP; e += DFM_NT) {
    const int i = e / NEWS_TP, t = e - i * NEWS_TP;
    Ms[e] = (i < ni && t < nt) ? (int)mask[(size_t)(i0 + i) * nr + t0 + t] : 0;
  }
  for (int t = DFM_TID; t < NEWS_TP; t += DFM_NT) Rp[t] = (t < nt) ? rowp_[(size_t)b * nr + t0 + t] : -1;
  DFM_SYNC();
  wt_gemm(Fsh, ld, 1, Ls, ld, 1, nt, ni, r, [&](int t, int i, double v) { Is[i * ldc + t] = v; });          // E[x | old]
  DFM_SYNC();
  for (int e = DFM_TID; e < ni * NEWS_TP; e += DFM_NT) {
    const int i = e / NEWS_TP, t = e - i * NEWS_TP;
    if (t >= nt) continue;
    const double v = Ms[e] ? Xn[((size_t)b * N + i0 + i) * ldn + row0 + t0 + t] - Is[i * ldc + t] : DFM_NAN;
    Is[i * ldc + t] = v;
    if (news) news[(size_t)b * onr + (size_t)(i0 + i) * nr + t0 + t] = v;
  }
  for (int q0 = 0; q0 < nq; q0 += NEWS_QC) {
    const int nqc = (nq - q0 < NEWS_QC) ? nq - q0 : NEWS_QC;
    DFM_SYNC();
    for (int e = DFM_TID; e < nqc * NEWS_TP * r; e += DFM_NT) {
      const int c = e % r, m = e / r, t = m % NEWS_TP, qq = m / NEWS_TP;
      const int a = Rp[t];
      Gs[m * ld + c] = (a >= 0) ? gv[(size_t)(q0 + qq) * nmax + a * r + c] : 0.0;
    }
    DFM_SYNC();
    wt_gemm(Gs, ld, 1, Ls, ld, 1, nqc * NEWS_TP, ni, r, [&](int m, int i, double v) { Wt[i * ldw + m] = v; });   // g' lam_i
    DFM_SYNC();
    for (int qq = 0; qq < nqc; ++qq) {
      const int q = q0 + qq, kd = kind_[(size_t)b * nq + q], ts = tser[q], tt = tper[q];
      double s = 0.0;
      for (int e = DFM_TID; e < ni * NEWS_TP; e += DFM_NT) {
        const int i = e / NEWS_TP, t = e - i * NEWS_TP;
        if (t >= nt) continue;
        double w = 0.0, c = 0.0;
        if (Ms[e]) {
          if (kd == NEWS_MODEL) w = Wt[i * ldw + qq * NEWS_TP + t] / Rs[i];
          else if (kd == NEWS_RELEASED) w = (i0 + i == ts && w0 + t0 + t == tt) ? 1.0 : 0.0;
          else if (kd == NEWS_OUT) w = DFM_NAN;
          c = w * Is[i * ldc + t];
        }
        s += c;
        const size_t g = ((size_t)b * nq + q) * onr + (size_t)(i0 + i) * nr + t0 + t;
        if (weight) weight[g] = w;
        if (contrib) contrib[g] = c;
      }
      s = block_sum(s, red);
      if (DFM_TID == 0) part[((size_t)b * ntile + tile) * nq + q] = s;
    }
  }
}

// new_est = old_est + the tiles' partial sums in tile order; NaN for a failed pair.  grid (B), 64 threads.
__global__ void k_news_finish(const double* __restrict__ part, int ntile, const double* __restrict__ oldv, const int* __restrict__ pstat,
                              int nq, double* __restrict__ old_est, double* __restrict__ new_est) {
  const int b = DFM_BX;
  const bool failed = pstat[b] != 0;
  for (int q = DFM_TID; q < nq; q += DFM_NT) {
    double o = DFM_NAN, v = DFM_NAN;
    if (!failed) {
      double s = 0.0;
      for (int j = 0; j < ntile; ++j) s += part[((size_t)b * ntile + j) * nq + q];
      o = oldv[(size_t)b * nq + q];
      v = o + s;
    }
    if (old_est) old_est[(size_t)b * nq + q] = o;
    if (new_est) new_est[(size_t)b * nq + q] = v;
  }
}

}  // namespace dfm
