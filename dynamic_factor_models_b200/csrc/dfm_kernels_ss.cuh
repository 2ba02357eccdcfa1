// dfm_kernels_ss.cuh -- smoothing, nowcasting and forecasting at FIXED parameters (dfm_kalman_smooth).
// The E-step is the general path's (k_em_contract / k_em_contract_bal -> k_em_filter_smooth) run once on panels padded
// with H all-missing periods: a forecast period is a period in which no series is observed, so the filter predicts
// through it and the smoother returns E[z_{T+h} | x] and its covariance.  This file holds the staging of the padded
// panels and the projection onto the series (common component, imputed values and their variances); the spec is
// smooth_forecast() in tests/forecast_oracle.py.
#pragma once
#include "dfm_common.cuh"
#include "dfm_kernels_em.cuh"

namespace dfm {

// Padded panel: Xp (Tp x cols, column-major) = [X; NaN (Tp - T rows)].  X == nullptr: only the NaN tail is written (the
// in-sample rows were copied already, e.g. by a strided host-to-device copy).  grid (ceil(cols / 8)), 256 threads.
__global__ void k_ss_pad(const double* __restrict__ X, int T, int Tp, long long cols, double* __restrict__ Xp) {
  const int t0 = X ? 0 : T;
  const int per = Tp - t0;
  for (long long e = (long long)DFM_BX * DFM_NT + DFM_TID; e < cols * per; e += (long long)DFM_GX * DFM_NT) {
    const long long c = e / per;
    const int t = t0 + (int)(e - c * per);
    Xp[c * Tp + t] = (t < T) ? X[c * T + t] : DFM_NAN;
  }
}

// Panels whose E-step failed (status 3: a covariance that is not positive definite, or R_i <= 0) return NaN factors,
// covariances and log-likelihood.  grid (B), one block.
__global__ void k_ss_nan_failed(const EmState* st, int T, int r, double* __restrict__ Fs, double* __restrict__ PsF,
                                double* __restrict__ ll) {
  const int b = DFM_BX;
  if (st[b].status != 3) return;
  const int np = r * (r + 1) / 2;
  for (long long e = DFM_TID; e < (long long)T * r; e += DFM_NT) Fs[(size_t)b * T * r + e] = DFM_NAN;
  for (long long e = DFM_TID; e < (long long)T * np; e += DFM_NT) PsF[(size_t)b * T * np + e] = DFM_NAN;
  if (DFM_TID == 0) ll[b] = DFM_NAN;
}

#define SS_TP 32               // periods per tile
#define SS_NS 64               // series per tile

__host__ __device__ inline size_t ss_project_smem_doubles(int r) {
  const size_t ld = (size_t)em_lds(r);
  return (size_t)SS_NS * ld + (size_t)SS_TP * ld + (size_t)r * r + (size_t)SS_NS * ld + 2 * (size_t)SS_NS * (SS_TP + 1) + SS_NS + SS_TP;
}

// Projection of the smoothed factors onto the series of one tile of SS_TP periods x SS_NS series of one panel:
//   common_it = lam_i' E[f_t | x]                  (F Lam' as DMMA tile products)
//   xhat_it   = x_it where observed, common_it otherwise
//   xvar_it   = 0 where observed, lam_i' PF_t lam_i + R_i otherwise,  the quadratic forms as rowsum((Lam PF_t) o Lam) with
//               Lam PF_t on the tensor path -- only for periods whose smoothed covariance differs from the previous
//               period's: inside a frozen run (the smoother's steady state) the row of the previous period is reused.
// Fs [Tp x r], PsF packed [Tp x np] per panel (k_em_filter_smooth), X the padded panel [Tp x N].  Series with a NaN
// loading or R_i are out of the model: NaN in every output; so is a whole panel whose status is 3.  Outputs may be NULL
// (not computed).  grid (ceil(Tp / SS_TP), ceil(N / SS_NS) * nb), 256 threads; panels b0 .. b0 + nb - 1.
__global__ void k_ss_project(const double* __restrict__ Xall, const double* __restrict__ Fs_, const double* __restrict__ PsF_,
                             const double* __restrict__ LamAll, const double* __restrict__ Rall, const EmState* st, int Tp, int N,
                             int r, int b0, double* __restrict__ common, double* __restrict__ xhat, double* __restrict__ xvar) {
  DFM_SMEM(sm);
  const int nst = (N + SS_NS - 1) / SS_NS;
  const int b = b0 + DFM_BY / nst, i0 = (DFM_BY % nst) * SS_NS, t0 = DFM_BX * SS_TP;
  const int ni = (N - i0 < SS_NS) ? N - i0 : SS_NS, nt = (Tp - t0 < SS_TP) ? Tp - t0 : SS_TP;
  const int ld = em_lds(r), np = r * (r + 1) / 2, ldv = SS_TP + 1;
  double* Ls = sm;                                   // [SS_NS][ld]  loadings of the tile's series
  double* Fsh = Ls + (size_t)SS_NS * ld;             // [SS_TP][ld]  smoothed factors of the tile's periods
  double* Pf = Fsh + (size_t)SS_TP * ld;             // [r][r]       PF_t
  double* G = Pf + (size_t)r * r;                    // [SS_NS][ld]  Lam PF_t
  double* Cs = G + (size_t)SS_NS * ld;               // [SS_NS][ldv] common component
  double* Vs = Cs + (size_t)SS_NS * ldv;             // [SS_NS][ldv] lam' PF_t lam + R
  double* Rs = Vs + (size_t)SS_NS * ldv;             // [SS_NS]
  int* newp = (int*)(Rs + SS_NS);                    // [SS_TP]      does PF_t differ from PF_{t-1}?
  const double* Lam = LamAll + (size_t)b * N * r; const double* R = Rall + (size_t)b * N;
  const double* Fs = Fs_ + (size_t)b * Tp * r; const double* PsF = PsF_ + (size_t)b * Tp * np;
  const double* X = Xall + (size_t)b * Tp * N;
  const bool failed = st[b].status == 3;
  for (int e = DFM_TID; e < SS_NS * r; e += DFM_NT) {
    const int i = e % SS_NS, a = e / SS_NS;
    Ls[i * ld + a] = (i < ni) ? Lam[i0 + i + (size_t)N * a] : 0.0;
  }
  for (int i = DFM_TID; i < SS_NS; i += DFM_NT) Rs[i] = (i < ni) ? R[i0 + i] : 0.0;
  for (int e = DFM_TID; e < SS_TP * r; e += DFM_NT) {
    const int t = e % SS_TP, a = e / SS_TP;
    Fsh[t * ld + a] = (t < nt) ? Fs[t0 + t + (size_t)Tp * a] : 0.0;
  }
  for (int t = DFM_TID; t < SS_TP; t += DFM_NT) newp[t] = (t == 0) ? 1 : 0;
  DFM_SYNC();
  if (xvar)                                          // (period, packed element) pairs over all threads: independent loads
    for (int e = DFM_TID; e < nt * np; e += DFM_NT) {
      const int t = e % nt, q = e / nt;
      if (t > 0 && PsF[t0 + t + (size_t)Tp * q] != PsF[t0 + t - 1 + (size_t)Tp * q]) newp[t] = 1;     // (benign race: all store 1)
    }
  DFM_SYNC();
  if (common || xhat)
    wt_gemm(Fsh, ld, 1, Ls, ld, 1, nt, ni, r, [&](int t, int i, double v) { Cs[i * ldv + t] = v; });
  if (xvar) {
    for (int t = 0; t < nt; ++t) {
      if (!newp[t]) {                                // frozen: the quadratic forms of the previous period
        for (int i = DFM_TID; i < ni; i += DFM_NT) Vs[i * ldv + t] = Vs[i * ldv + t - 1];
        continue;
      }
      for (int e = DFM_TID; e < r * r; e += DFM_NT) {
        const int a = e % r, c = e / r;
        Pf[e] = PsF[t0 + t + (size_t)Tp * ((a >= c) ? pidx(a, c) : pidx(c, a))];
      }
      DFM_SYNC();
      wt_gemm(Ls, ld, 1, Pf, r, 1, ni, r, r, [&](int i, int c, double v) { G[i * ld + c] = v; });     // Lam PF_t
      DFM_SYNC();
      for (int i = DFM_TID; i < ni; i += DFM_NT) {
        double s0 = 0.0, s1 = 0.0;
        int a = 0;
        for (; a + 1 < r; a += 2) { s0 += G[i * ld + a] * Ls[i * ld + a]; s1 += G[i * ld + a + 1] * Ls[i * ld + a + 1]; }
        if (a < r) s0 += G[i * ld + a] * Ls[i * ld + a];
        Vs[i * ldv + t] = (s0 + s1) + Rs[i];
      }
    }
  }
  DFM_SYNC();
  // coalesced write-out: consecutive threads take consecutive periods of one series
  for (int e = DFM_TID; e < ni * SS_TP; e += DFM_NT) {
    const int i = e / SS_TP, t = e - i * SS_TP;
    if (t >= nt) continue;
    const size_t g = (size_t)b * Tp * N + (size_t)(i0 + i) * Tp + t0 + t;
    const bool out = failed || is_nan(Ls[i * ld]) || is_nan(Rs[i]);
    const double c = out ? DFM_NAN : Cs[i * ldv + t];
    if (common) common[g] = c;
    if (xhat || xvar) {
      const double x = X[(size_t)(i0 + i) * Tp + t0 + t];
      const bool obs = !is_nan(x);
      if (xhat) xhat[g] = out ? DFM_NAN : (obs ? x : c);
      if (xvar) xvar[g] = out ? DFM_NAN : (obs ? 0.0 : Vs[i * ldv + t]);
    }
  }
}

}  // namespace dfm
