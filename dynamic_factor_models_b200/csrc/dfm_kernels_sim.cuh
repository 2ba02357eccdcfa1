// dfm_kernels_sim.cuh -- the simulation smoother (dfm_simulation_smoother): draws of the factor path and of the missing cells
// from their JOINT posterior given the observed cells, at fixed state-space parameters (Durbin & Koopman 2002, mean-corrected
// form).  The spec is tests/simsmooth_oracle.py.  After the fixed-parameter E-step of dfm_kalman_smooth (same kernels, same
// scratch) three kernels run:
//   k_sim_gains    one CTA per period: the draw-independent matrices of the two mean recursions, from P_{t|t} = Pf[src[t]],
//                  P_{t+1|t} = Pp[src[t+1]] and C_t (no recurrence between periods, so frozen periods simply recompute)
//   k_sim_paths    SIM_ND draws per CTA: the unconditional state z+ and the filter on c_t = b_t - C_t f+_t - L_C,t xi_t
//                  forward, the RTS smoother backward; every product is a DMMA tile product (wt_gemm) with the draws'
//                  state tile [SIM_ND x k] as the n operand
//   k_sim_project  tiles of periods x series x draws: x~ = the data where observed, lam_i' f~_t + sqrt(R_i) eps_it where
//                  missing (F~ Lam' as DMMA tile products); bound by its HBM writes
// A draw costs O(Tp k^2), not O(Tp N r): the information of x - x+ is formed from b_t directly, because
// b_t(x+) = C_t f+_t + sum_{i obs} lam_i e+_it / R_i and the sum is N(0, C_t), independent of everything else.
// Normals: rng_normal(seed, draw id, stream, element) (dfm_kernels_rep.cuh) on four streams:
//   RNG_SS_Z0    nu      z+_0 = L_P0 nu                          element a           (a < k)
//   RNG_SS_ETA   eta_t   z+_t = M z+_{t-1} + E' L_Q eta_t, t >= 1  element t r + a     (a < r)
//   RNG_SS_OBS   xi_t    the N(0, C_t) term of c_t              element t r + a     (a < r)
//   RNG_SS_MISS  eps_it  idiosyncratic draw of a missing cell   element i Tp + t    (drawn for missing cells only)
// so draw d is a pure function of (seed, d): any split of a draw range over calls or GPUs gives bit-identical draws.
#pragma once
#include "dfm_common.cuh"
#include "dfm_kernels_em.cuh"
#include "dfm_kernels_rep.cuh"
#include "dfm_kernels_ss.cuh"

namespace dfm {

enum { RNG_SS_Z0 = 7, RNG_SS_ETA = 8, RNG_SS_OBS = 9, RNG_SS_MISS = 10 };

#define SIM_ND 16              // draws per CTA of k_sim_paths
#define SIM_NT 128             // threads per CTA of k_sim_paths
#define SIM_PD 8               // draws per CTA of k_sim_project
#define SIM_PIVOT_TOL 1e-12    // a Cholesky pivot <= SIM_PIVOT_TOL * max diag counts as zero

// Gain table, per period t (stride sim_gain_stride):
//   G_t = [Phi_t | -K_t C_t | -K_t L_C,t]   k x (k + 2r)   Phi_t = (I - K_t C_t E) M,  K_t = Pf_t E'
//   kb_t = K_t b_t                           k
//   H_t = [I - J_t M | J_t]                  k x 2k         J_t = Pf_t M' Pp_{t+1}^-1  (t = Tp - 1: [I | 0])
// so that zf_t = G_t [zf_{t-1}; f+_t; xi_t] + kb_t and zs_t = H_t [zf_t; zs_{t+1}].  After the Tp periods: L_P0 (k x k),
// then [A | L_Q] (r x (k + r)).  All column-major.
__host__ __device__ inline size_t sim_gain_stride(int k, int r) { return (size_t)k * (k + 2 * r) + k + 2 * (size_t)k * k; }
__host__ __device__ inline size_t sim_gains_doubles(int Tp, int k, int r) {
  return (size_t)Tp * sim_gain_stride(k, r) + (size_t)k * k + (size_t)r * (k + r);
}

// In-place lower Cholesky factor of the n x n PSD matrix A (lower triangle read, upper triangle zeroed), unpivoted; a pivot
// <= SIM_PIVOT_TOL * max_i A_ii zeroes its column and the elimination continues (C_t = 0 in forecast periods, rank-deficient
// C_t where fewer than r series are observed, a singular P0).  The pivot decisions are the oracle's psd_cholesky.
__device__ inline void bm_chol_psd(double* A, int ld, int n) {
  double dmax = 0.0;
  for (int j = 0; j < n; ++j) dmax = fmax(dmax, A[j + ld * j]);
  const double tol = SIM_PIVOT_TOL * dmax;
  for (int j = 0; j < n; ++j) {
    const double d = A[j + ld * j];
    DFM_SYNC();                                        // (everyone has read the pivot)
    if (d > tol) {
      const double s = sqrt(d);
      for (int i = j + DFM_TID; i < n; i += DFM_NT) A[i + ld * j] = (i == j) ? s : A[i + ld * j] / s;
      DFM_SYNC();
      const int m = n - j - 1;
      for (int e = DFM_TID; e < m * m; e += DFM_NT) {
        const int i = j + 1 + e % m, c = j + 1 + e / m;
        if (i >= c) A[i + ld * c] -= A[i + ld * j] * A[c + ld * j];
      }
    } else {
      for (int i = j + DFM_TID; i < n; i += DFM_NT) A[i + ld * j] = 0.0;
    }
    DFM_SYNC();
  }
  for (int e = DFM_TID; e < n * n; e += DFM_NT) { const int i = e % n, j = e / n; if (i < j) A[i + ld * j] = 0.0; }
  DFM_SYNC();
}

__host__ __device__ inline size_t sim_gains_smem_doubles(int r, int p) {
  const size_t k = (size_t)r * p;
  return 5 * k * k + 2 * (size_t)r * r + 2 * (size_t)r * k + 8;
}

// The gain table of one model from the E-step of k_em_filter_smooth over Tp periods: Pp / Pf at the explicit periods and
// src[t] (the period whose covariances period t uses), b_t (Bt), the packed C_t (Ct) when the panel has missing cells, else
// the constant C, and n_t (nobs).  The E-step forms C_t as C minus the missing series' terms, which leaves rounding noise
// (~1e-16 |C|) where nothing is observed; its square root would be ~1e-8 |C|^1/2, so C_t of a period with n_t = 0 (a forecast
// period) is taken as exactly 0.  status: 0 on entry; set to the E-step's status, or to 3 if some P_{t+1|t} is not positive
// definite.
// grid (Tp + 1, models): CTA t < Tp builds period t, CTA Tp the period-independent factors.  Model c = DFM_BY of a batch of
// E-steps (dfm_gibbs: one model per chain) reads and writes at the per-model strides of the E-step's buffers (A r x k, Q and C
// r x r, P0 k x k, Ct Tp x r(r+1)/2, Bt Tp x r, Pp / Pf Tp x k x k, src / nobs Tp, st 1) and of the gain table
// (sim_gains_doubles), and status[c]; one model (grid.y = 1) is dfm_simulation_smoother's call.
__global__ void k_sim_gains(const double* __restrict__ A, const double* __restrict__ Q, const double* __restrict__ P0,
                            const double* __restrict__ Cg, const double* __restrict__ Ct, const double* __restrict__ Bt,
                            const double* __restrict__ Ppg, const double* __restrict__ Pfg, const int* __restrict__ src,
                            const int* __restrict__ nobs, const EmState* st, int Tp, int r, int p, double* __restrict__ gains,
                            int* status) {
  DFM_SMEM(sm);
  const int t = DFM_BX, k = r * p, kk = k * k, rr = r * r, rk = r * k;
  if (DFM_BY > 0) {
    const size_t c = DFM_BY;
    A += c * rk; Q += c * rr; P0 += c * kk; Cg += c * rr; Ct += c * Tp * (size_t)(r * (r + 1) / 2); Bt += c * Tp * r;
    Ppg += c * Tp * kk; Pfg += c * Tp * kk; src += c * Tp; nobs += c * Tp; st += c; gains += c * sim_gains_doubles(Tp, k, r);
    status += c;
  }
  if (st->status != 0) { if (DFM_TID == 0) atomicMax(status, st->status); return; }
  double* M = sm;      double* Pf = M + kk;   double* Pp = Pf + kk;  double* T1 = Pp + kk;  double* T2 = T1 + kk;
  double* Cs = T2 + kk; double* LC = Cs + rr; double* KC = LC + rr;  double* KL = KC + rk;
  int* info = (int*)(KL + rk);
  for (int e = DFM_TID; e < kk; e += DFM_NT) {
    const int i = e % k, j = e / k;
    M[e] = (i < r) ? A[i + r * j] : ((j == i - r) ? 1.0 : 0.0);
  }
  if (t == Tp) {                                       // L_P0 and [A | L_Q]
    double* g = gains + (size_t)Tp * sim_gain_stride(k, r);
    for (int e = DFM_TID; e < kk; e += DFM_NT) T1[e] = P0[e];
    for (int e = DFM_TID; e < rr; e += DFM_NT) Cs[e] = Q[e];
    DFM_SYNC();
    bm_chol_psd(T1, k, k);
    bm_chol_psd(Cs, r, r);
    for (int e = DFM_TID; e < kk; e += DFM_NT) g[e] = T1[e];
    for (int e = DFM_TID; e < r * (k + r); e += DFM_NT) { const int i = e % r, j = e / r; g[kk + e] = (j < k) ? A[i + r * j] : Cs[i + r * (j - k)]; }
    return;
  }
  const int hm = st->has_missing, none = nobs[t] == 0;
  const int sf = src[t];
  for (int e = DFM_TID; e < kk; e += DFM_NT) Pf[e] = Pfg[(size_t)sf * kk + e];
  for (int e = DFM_TID; e < rr; e += DFM_NT) {
    const int a = e % r, c = e / r;
    const double v = none ? 0.0 : hm ? Ct[t + (size_t)Tp * ((a >= c) ? pidx(a, c) : pidx(c, a))] : Cg[e];
    Cs[e] = v; LC[e] = v;
  }
  if (DFM_TID == 0) info[0] = 0;
  DFM_SYNC();
  bm_chol_psd(LC, r, r);
  double* G = gains + (size_t)t * sim_gain_stride(k, r);
  double* kb = G + (size_t)k * (k + 2 * r);
  double* Hm = kb + k;
  bm_gemm(KC, k, Pf, k, false, Cs, r, false, k, r, r, 1.0, 0.0);          // K C    (K = Pf[:, 0:r])
  bm_gemm(KL, k, Pf, k, false, LC, r, false, k, r, r, 1.0, 0.0);          // K L_C
  for (int e = DFM_TID; e < kk; e += DFM_NT) G[e] = M[e];
  DFM_SYNC();
  bm_gemm(G, k, KC, k, false, A, r, false, k, k, r, -1.0, 1.0);          // Phi = M - K C A   (E M = A)
  for (int e = DFM_TID; e < rk; e += DFM_NT) { G[kk + e] = -KC[e]; G[kk + rk + e] = -KL[e]; }
  for (int i = DFM_TID; i < k; i += DFM_NT) {
    double s = 0.0;
    for (int a = 0; a < r; ++a) s += Pf[i + k * a] * Bt[t + (size_t)Tp * a];
    kb[i] = s;
  }
  if (t + 1 < Tp) {
    const int sp = src[t + 1];
    for (int e = DFM_TID; e < kk; e += DFM_NT) Pp[e] = Ppg[(size_t)sp * kk + e];
    DFM_SYNC();
    bm_gemm(T1, k, M, k, false, Pf, k, false, k, k, k, 1.0, 0.0);         // M Pf
    bm_chol(Pp, k, k, info);
    bm_trsm_lower(Pp, k, k, T1, k, k);
    bm_trsm_lowerT(Pp, k, k, T1, k, k);                                   // Pp^-1 M Pf = J'
    if (DFM_TID == 0 && info[0]) atomicMax(status, 3);
    for (int e = DFM_TID; e < kk; e += DFM_NT) { const int i = e % k, j = e / k; Hm[kk + e] = T1[j + k * i]; }
    bm_gemm(Hm, k, T1, k, true, M, k, false, k, k, k, -1.0, 0.0);         // -J M
    for (int i = DFM_TID; i < k; i += DFM_NT) Hm[i + k * i] += 1.0;
  } else {
    for (int e = DFM_TID; e < 2 * kk; e += DFM_NT) { const int i = e % k, j = e / k; Hm[e] = (i == j) ? 1.0 : 0.0; }
  }
}

__host__ __device__ inline size_t sim_paths_smem_doubles(int r, int p) {
  const int k = r * p;
  const size_t g1 = (size_t)k * (k + 2 * r), g2 = 2 * (size_t)k * k;
  const size_t fw = (size_t)em_lds(k + r) + em_lds(k + 2 * r), bw = (size_t)em_lds(2 * k);
  return (g1 > g2 ? g1 : g2) + (size_t)k * k + (size_t)r * (k + r) + k + 2 * SIM_ND * (fw > bw ? fw : bw);
}

// The factor draws of draws id0 .. id0 + nd - 1 (one chunk): SIM_ND draws per CTA, SIM_NT threads.
// Forward:  z+_0 = L_P0 nu, z+_t = [A | L_Q] [z+_{t-1}; eta_t] on top of the shifted lags;  zf_t = G_t [zf_{t-1}; f+_t; xi_t]
//           + kb_t.  zf_t and f+_t go to the chunk's scratch zfS [Tp][nd][k], fS [Tp][nd][r].
// Backward: zs_{Tp-1} = zf_{Tp-1},  zs_t = H_t [zf_t; zs_{t+1}];  f~_t = f+_t + E zs_t overwrites f+_t in fS and goes to
//           Fout[d] (Tp x r column-major per draw; may be NULL).
// The gains are copied to shared memory only when src changes (a frozen period's matrices are its source period's).
// status != 0 (failed E-step): NaN factor draws.
__global__ void k_sim_paths(const double* __restrict__ gains, const int* __restrict__ src, int Tp, int r, int p,
                            unsigned long long seed, long long id0, int nd, const int* __restrict__ status,
                            double* __restrict__ zfS, double* __restrict__ fS, double* __restrict__ Fout) {
  DFM_SMEM(sm);
  const int k = r * p, kk = k * k, kr2 = k + 2 * r;
  const size_t gstr = sim_gain_stride(k, r);
  const int ldp = em_lds(k + r), ldw = em_lds(kr2), ldy = em_lds(2 * k);
  const int j0 = DFM_BX * SIM_ND, nv = (nd - j0 < SIM_ND) ? nd - j0 : SIM_ND;
  if (*status != 0) {
    if (Fout) for (long long e = DFM_TID; e < (long long)nv * Tp * r; e += DFM_NT) Fout[(size_t)j0 * Tp * r + e] = DFM_NAN;
    return;
  }
  const size_t g1 = (size_t)k * kr2, g2 = 2 * (size_t)kk;
  const size_t fw = (size_t)ldp + ldw, bw = (size_t)ldy;
  double* Gs = sm;                                     // G_t (forward) / H_t (backward)
  double* LP0 = Gs + (g1 > g2 ? g1 : g2);
  double* AQ = LP0 + kk;                               // [A | L_Q]
  double* kb = AQ + (size_t)r * (k + r);
  double* rows = kb + k;                               // forward: Pz[2][SIM_ND][ldp], Wz[2][SIM_ND][ldw]; backward: Y[2][SIM_ND][ldy]
  double* Pz[2] = {rows, rows + SIM_ND * ldp};                           // [z+ | eta]
  double* Wz[2] = {rows + 2 * SIM_ND * ldp, rows + 2 * SIM_ND * ldp + SIM_ND * ldw};   // [zf_{t-1} | f+_t | xi_t]
  const double* gtail = gains + (size_t)Tp * gstr;
  const unsigned long long idb = (unsigned long long)(id0 + j0);
  for (int e = DFM_TID; e < kk; e += DFM_NT) LP0[e] = gtail[e];
  for (int e = DFM_TID; e < r * (k + r); e += DFM_NT) AQ[e] = gtail[kk + e];
  for (size_t e = DFM_TID; e < 2 * SIM_ND * (fw > bw ? fw : bw); e += DFM_NT) rows[e] = 0.0;
  DFM_SYNC();
  for (int e = DFM_TID; e < nv * k; e += DFM_NT) { const int n = e / k, a = e - n * k; Pz[1][n * ldp + a] = rng_normal(seed, idb + n, RNG_SS_Z0, a); }
  // ------------------------------------------------------------------ forward
  int gsrc = -1;
  for (int t = 0; t < Tp; ++t) {
    double* Pc = Pz[t & 1];        // z+_t
    double* Pq = Pz[(t + 1) & 1];  // [z+_{t-1} | eta_t]  (t = 0: nu)
    double* Wc = Wz[t & 1];
    double* Wn = Wz[(t + 1) & 1];
    for (int e = DFM_TID; e < nv * r; e += DFM_NT) {
      const int n = e / r, a = e - n * r;
      if (t > 0) Pq[n * ldp + k + a] = rng_normal(seed, idb + n, RNG_SS_ETA, (unsigned long long)t * r + a);
      Wc[n * ldw + k + r + a] = rng_normal(seed, idb + n, RNG_SS_OBS, (unsigned long long)t * r + a);
    }
    const double* gt = gains + (size_t)t * gstr;
    if (src[t] != gsrc) { for (int e = DFM_TID; e < k * kr2; e += DFM_NT) Gs[e] = gt[e]; gsrc = src[t]; }
    for (int e = DFM_TID; e < k; e += DFM_NT) kb[e] = gt[(size_t)k * kr2 + e];
    DFM_SYNC();
    if (t == 0) {
      wt_gemm(LP0, 1, k, Pq, ldp, 1, k, nv, k, [&](int i, int n, double v) { Pc[n * ldp + i] = v; });
    } else {
      wt_gemm(AQ, 1, r, Pq, ldp, 1, r, nv, k + r, [&](int a, int n, double v) { Pc[n * ldp + a] = v; });
      for (int e = DFM_TID; e < nv * (k - r); e += DFM_NT) { const int n = e / (k - r), i = e - n * (k - r); Pc[n * ldp + r + i] = Pq[n * ldp + i]; }
    }
    DFM_SYNC();
    for (int e = DFM_TID; e < nv * r; e += DFM_NT) {
      const int n = e / r, a = e - n * r;
      const double v = Pc[n * ldp + a];
      Wc[n * ldw + k + a] = v;
      fS[((size_t)t * nd + j0 + n) * r + a] = v;
    }
    DFM_SYNC();
    wt_gemm(Gs, 1, k, Wc, ldw, 1, k, nv, kr2, [&](int i, int n, double v) {
      v += kb[i];
      Wn[n * ldw + i] = v;
      zfS[((size_t)t * nd + j0 + n) * k + i] = v;
    });
    DFM_SYNC();
  }
  // ------------------------------------------------------------------ backward
  double* Y[2] = {rows, rows + SIM_ND * ldy};          // Y[t & 1] = [zf_t | zs_{t+1}]
  {
    const int t = Tp - 1;
    double* Yl = Y[(t - 1) & 1];
    for (int e = DFM_TID; e < nv * k; e += DFM_NT) {
      const int n = e / k, i = e - n * k;
      const double v = zfS[((size_t)t * nd + j0 + n) * k + i];
      Yl[n * ldy + k + i] = v;
      if (i < r) {
        const size_t o = ((size_t)t * nd + j0 + n) * r + i;
        const double f = fS[o] + v;
        fS[o] = f;
        if (Fout) Fout[(size_t)(j0 + n) * Tp * r + t + (size_t)Tp * i] = f;
      }
    }
  }
  int hs0 = -1, hs1 = -1;
  for (int t = Tp - 2; t >= 0; --t) {
    double* Yc = Y[t & 1];
    double* Yn = Y[(t + 1) & 1];                       // receives zs_t (the next step's operand)
    for (int e = DFM_TID; e < nv * k; e += DFM_NT) { const int n = e / k, i = e - n * k; Yc[n * ldy + i] = zfS[((size_t)t * nd + j0 + n) * k + i]; }
    if (src[t] != hs0 || src[t + 1] != hs1) {
      const double* ht = gains + (size_t)t * gstr + (size_t)k * kr2 + k;
      for (int e = DFM_TID; e < 2 * kk; e += DFM_NT) Gs[e] = ht[e];
      hs0 = src[t]; hs1 = src[t + 1];
    }
    DFM_SYNC();
    wt_gemm(Gs, 1, k, Yc, ldy, 1, k, nv, 2 * k, [&](int i, int n, double v) {
      Yn[n * ldy + k + i] = v;
      if (i < r) {
        const size_t o = ((size_t)t * nd + j0 + n) * r + i;
        const double f = fS[o] + v;
        fS[o] = f;
        if (Fout) Fout[(size_t)(j0 + n) * Tp * r + t + (size_t)Tp * i] = f;
      }
    });
    DFM_SYNC();
  }
}

__host__ __device__ inline size_t sim_project_smem_doubles(int r) {
  const size_t ld = (size_t)em_lds(r);
  return (size_t)SS_NS * ld + (size_t)SS_TP * ld + 2 * (size_t)SS_NS * (SS_TP + 1) + SS_NS;
}

// Panel draws of one chunk: tile of SS_TP periods x SS_NS series x SIM_PD draws.  X: the padded panel (Tp x N); fS: the
// factor draws [Tp][nd][r] of k_sim_paths; Xout[d]: Tp x N column-major per draw.  The data where observed,
// lam_i' f~_t + sqrt(R_i) eps_it where missing, NaN for a series out of the model and everywhere when status != 0.  Writes
// are staged through shared memory so that consecutive threads store consecutive periods of one series.
// pstride = 0: one model (Lam, R, *status) for every draw, draw j has id id0 + j (dfm_simulation_smoother).  pstride = 1: draw j
// has its own model (Lam + j N r, R + j N, status[j]) and id id0 + j idstride (dfm_gibbs: one draw per chain).
// grid (ceil(Tp / SS_TP), ceil(N / SS_NS) * ceil(nd / SIM_PD)), 256 threads.
__global__ void k_sim_project(const double* __restrict__ X, const double* __restrict__ Lam, const double* __restrict__ R,
                              const double* __restrict__ fS, int Tp, int N, int r, unsigned long long seed, long long id0, int nd,
                              const int* __restrict__ status, double* __restrict__ Xout, int pstride, long long idstride) {
  DFM_SMEM(sm);
  const int nst = (N + SS_NS - 1) / SS_NS;
  const int i0 = (DFM_BY % nst) * SS_NS, d0 = (DFM_BY / nst) * SIM_PD, t0 = DFM_BX * SS_TP;
  const int ni = (N - i0 < SS_NS) ? N - i0 : SS_NS, nt = (Tp - t0 < SS_TP) ? Tp - t0 : SS_TP;
  const int dn = (nd - d0 < SIM_PD) ? nd - d0 : SIM_PD;
  const int ld = em_lds(r), ldv = SS_TP + 1;
  double* Ls = sm;                                     // [SS_NS][ld]   loadings of the tile's series
  double* Fsh = Ls + (size_t)SS_NS * ld;               // [SS_TP][ld]   one draw's factors of the tile's periods
  double* Xs = Fsh + (size_t)SS_TP * ld;               // [SS_NS][ldv]  the data
  double* Cs = Xs + (size_t)SS_NS * ldv;               // [SS_NS][ldv]  lam_i' f~_t
  double* Sd = Cs + (size_t)SS_NS * ldv;               // [SS_NS]       sqrt(R_i), NaN for a series out of the model
  bool failed = *status != 0;
  auto load_model = [&](const double* Lm, const double* Rm) {
    for (int e = DFM_TID; e < SS_NS * r; e += DFM_NT) {
      const int i = e % SS_NS, a = e / SS_NS;
      Ls[i * ld + a] = (i < ni) ? Lm[i0 + i + (size_t)N * a] : 0.0;
    }
    for (int i = DFM_TID; i < SS_NS; i += DFM_NT) Sd[i] = (i < ni && !is_nan(Lm[i0 + i])) ? sqrt(Rm[i0 + i]) : DFM_NAN;
  };
  if (!pstride) load_model(Lam, R);
  for (int e = DFM_TID; e < ni * SS_TP; e += DFM_NT) {
    const int i = e / SS_TP, t = e - i * SS_TP;
    if (t < nt) Xs[i * ldv + t] = X[(size_t)(i0 + i) * Tp + t0 + t];
  }
  for (int d = 0; d < dn; ++d) {
    const int j = d0 + d;
    const unsigned long long id = pstride ? (unsigned long long)(id0 + (long long)j * idstride) : (unsigned long long)(id0 + j);
    DFM_SYNC();
    if (pstride) {
      load_model(Lam + (size_t)j * N * r, R + (size_t)j * N);
      failed = status[j] != 0;
    }
    for (int e = DFM_TID; e < nt * r; e += DFM_NT) { const int t = e / r, a = e - t * r; Fsh[t * ld + a] = fS[((size_t)(t0 + t) * nd + j) * r + a]; }
    DFM_SYNC();
    wt_gemm(Fsh, ld, 1, Ls, ld, 1, nt, ni, r, [&](int t, int i, double v) { Cs[i * ldv + t] = v; });
    DFM_SYNC();
    double* xo = Xout + (size_t)j * Tp * N;
    for (int e = DFM_TID; e < ni * SS_TP; e += DFM_NT) {
      const int i = e / SS_TP, t = e - i * SS_TP;
      if (t >= nt) continue;
      const double x = Xs[i * ldv + t], sd = Sd[i];
      double v;
      if (failed || is_nan(sd)) v = DFM_NAN;
      else if (!is_nan(x)) v = x;
      else v = Cs[i * ldv + t] + sd * rng_normal(seed, id, RNG_SS_MISS, (unsigned long long)(i0 + i) * Tp + t0 + t);
      xo[(size_t)(i0 + i) * Tp + t0 + t] = v;
    }
  }
}

}  // namespace dfm
