// dfm_kernels_ssb.cuh -- parametric bootstrap of a fitted state-space DFM (dfm_ss_simulate_panels, dfm_ss_bootstrap).  The
// spec is tests/ss_bootstrap_oracle.py.
//   k_ss_sim_chol     once per call: L_P0 and [A | L_Q] of the fitted parameters (shared by every replicate)
//   k_ss_simulate     SSB_ND replicates per CTA: the state z_1 = L_P0 nu, z_t = M z_{t-1} + [L_Q eta_t; 0], every step a DMMA
//                     tile product (wt_gemm) with the replicates' state tile as the n operand and [A | L_Q] as the m operand;
//                     the factors f_t go to scratch [b][t][r]
//   k_ss_sim_project  tiles of periods x series x replicates: x_it = lam_i' f_t + sqrt(R_i) eps_it where the template panel is
//                     observed, NaN where it is missing or the series is out of the model (F Lam' as DMMA tile products); bound
//                     by its HBM writes
//   k_ss_align        one CTA per replicate: the re-estimated parameters brought back into the rotation of the fitted ones, and
//                     the companion form that dfm_irf takes
// Normals: rng_normal(seed, replication id, stream, element) (dfm_kernels_rep.cuh) on three streams (T periods, k = r p):
//   RNG_SSB_Z0   11  nu      z_1 = L_P0 nu                        element a          (a < k)
//   RNG_SSB_ETA  12  eta_t   state shocks of periods t >= 1       element t r + a    (a < r)
//   RNG_SSB_EPS  13  eps_it  idiosyncratic draw of a cell          element i T + t    (drawn for cells the template observes)
// Tags 0-6 are the replication generators', 7-10 the simulation smoother's.  Replicate b of a call is replication id rep0 + b,
// a pure function of (seed, rep0 + b): any split of a replication range over calls or GPUs gives bit-identical panels.
#pragma once
#include "dfm_common.cuh"
#include "dfm_kernels_rep.cuh"
#include "dfm_kernels_sim.cuh"
#include "dfm_kernels_ss.cuh"

namespace dfm {

enum { RNG_SSB_Z0 = 11, RNG_SSB_ETA = 12, RNG_SSB_EPS = 13 };

#define SSB_ND 8               // replicates per CTA of k_ss_simulate
#define SSB_NT 128             // threads per CTA of k_ss_simulate and k_ss_align
#define SSB_NC 64              // series per staged chunk of k_ss_align
#define SSB_SING_TOL 1e-12     // alignment: a pivot <= SSB_SING_TOL * (largest diagonal / largest entry) counts as singular

// g = [L_P0 (k x k) | [A | L_Q] (r x (k + r))], column-major; the PSD Cholesky factors of the simulation smoother
// (bm_chol_psd: a pivot <= 1e-12 max diag is a zero column).  grid (1).
__host__ __device__ inline size_t ssb_chol_doubles(int r, int p) { const size_t k = (size_t)r * p; return k * k + (size_t)r * (k + r); }
__host__ __device__ inline size_t ssb_chol_smem_doubles(int r, int p) { const size_t k = (size_t)r * p; return k * k + (size_t)r * r; }
__global__ void k_ss_sim_chol(const double* __restrict__ A, const double* __restrict__ Q, const double* __restrict__ P0, int r, int p,
                              double* __restrict__ g) {
  DFM_SMEM(sm);
  const int k = r * p, kk = k * k, rr = r * r;
  double* LP = sm; double* LQ = LP + kk;
  for (int e = DFM_TID; e < kk; e += DFM_NT) LP[e] = P0[e];
  for (int e = DFM_TID; e < rr; e += DFM_NT) LQ[e] = Q[e];
  DFM_SYNC();
  bm_chol_psd(LP, k, k);
  bm_chol_psd(LQ, r, r);
  for (int e = DFM_TID; e < kk; e += DFM_NT) g[e] = LP[e];
  for (int e = DFM_TID; e < r * (k + r); e += DFM_NT) { const int i = e % r, j = e / r; g[kk + e] = (j < k) ? A[i + r * j] : LQ[i + r * (j - k)]; }
}

__host__ __device__ inline size_t ssb_sim_smem_doubles(int r, int p) {
  const int k = r * p;
  return ssb_chol_doubles(r, p) + 2 * (size_t)SSB_ND * em_lds(k + r);
}

// Factor paths of replicates rep0 .. rep0 + nb - 1: SSB_ND per CTA, SSB_NT threads.  fS: [nb][T][r] (row t of replicate b at
// fS + (b T + t) r).  Pz[t & 1] receives [z_t | eta_{t+1}], Pz[(t + 1) & 1] is the operand [z_{t-1} | eta_t] (t = 0: nu).
// One barrier per period: the normals of period t + 1 are drawn, and the factors of period t - 1 stored, in the phase of the
// period-t product (disjoint addresses); the normals go to the highest threads first, the product's tiles to the lowest warps,
// so that with SSB_ND r <= SSB_NT / 2 the Philox / Box-Muller latency is off the serial chain of the recursion.
__global__ void k_ss_simulate(const double* __restrict__ g, int T, int r, int p, unsigned long long seed, long long rep0, int nb,
                              double* __restrict__ fS) {
  DFM_SMEM(sm);
  const int k = r * p, kk = k * k, ldp = em_lds(k + r);
  const int j0 = DFM_BX * SSB_ND, nv = (nb - j0 < SSB_ND) ? nb - j0 : SSB_ND;
  double* LP0 = sm;
  double* AQ = LP0 + kk;                               // [A | L_Q]
  double* rows = AQ + (size_t)r * (k + r);
  double* Pz[2] = {rows, rows + SSB_ND * ldp};
  const unsigned long long idb = (unsigned long long)(rep0 + j0);
  for (int e = DFM_TID; e < kk; e += DFM_NT) LP0[e] = g[e];
  for (int e = DFM_TID; e < r * (k + r); e += DFM_NT) AQ[e] = g[kk + e];
  for (int e = DFM_TID; e < 2 * SSB_ND * ldp; e += DFM_NT) rows[e] = 0.0;
  DFM_SYNC();
  for (int e = DFM_TID; e < nv * k; e += DFM_NT) { const int n = e / k, a = e - n * k; Pz[1][n * ldp + a] = rng_normal(seed, idb + n, RNG_SSB_Z0, a); }
  DFM_SYNC();
  for (int t = 0; t < T; ++t) {
    double* Pc = Pz[t & 1];
    double* Pq = Pz[(t + 1) & 1];
    if (t == 0) {
      wt_gemm(LP0, 1, k, Pq, ldp, 1, k, nv, k, [&](int i, int n, double v) { Pc[n * ldp + i] = v; });
    } else {
      wt_gemm(AQ, 1, r, Pq, ldp, 1, r, nv, k + r, [&](int a, int n, double v) { Pc[n * ldp + a] = v; });
      for (int e = DFM_TID; e < nv * (k - r); e += DFM_NT) { const int n = e / (k - r), i = e - n * (k - r); Pc[n * ldp + r + i] = Pq[n * ldp + i]; }
      for (int e = DFM_TID; e < nv * r; e += DFM_NT) {
        const int n = e / r, a = e - n * r;
        fS[((size_t)(j0 + n) * T + t - 1) * r + a] = Pq[n * ldp + a];
      }
    }
    if (t + 1 < T)                                     // (the last threads first: the warps of the product come last)
      for (int e = DFM_NT - 1 - DFM_TID; e < nv * r; e += DFM_NT) {
        const int n = e / r, a = e - n * r;
        Pc[n * ldp + k + a] = rng_normal(seed, idb + n, RNG_SSB_ETA, (unsigned long long)(t + 1) * r + a);
      }
    DFM_SYNC();
  }
  const double* Pl = Pz[(T - 1) & 1];
  for (int e = DFM_TID; e < nv * r; e += DFM_NT) {
    const int n = e / r, a = e - n * r;
    fS[((size_t)(j0 + n) * T + T - 1) * r + a] = Pl[n * ldp + a];
  }
}

__host__ __device__ inline size_t ssb_project_smem_doubles(int r) {
  const size_t ld = (size_t)em_lds(r);
  return (size_t)SS_NS * ld + (size_t)SS_TP * ld + (size_t)SS_NS * (SS_TP + 1) + SS_NS + (size_t)SS_NS * SS_TP;
}

// Panels of one call: tile of SS_TP periods x SS_NS series x SIM_PD replicates.  Xt: the template panel (T x N; only its NaN
// pattern is read); fS: the factors of k_ss_simulate; Xout: [nb][N][T] column-major panels.  Writes are staged through shared
// memory so that consecutive threads store consecutive periods of one series.
// grid (ceil(T / SS_TP), ceil(N / SS_NS) * ceil(nb / SIM_PD)), 256 threads.
__global__ void k_ss_sim_project(const double* __restrict__ Xt, const double* __restrict__ Lam, const double* __restrict__ R,
                                 const double* __restrict__ fS, int T, int N, int r, unsigned long long seed, long long rep0, int nb,
                                 double* __restrict__ Xout) {
  DFM_SMEM(sm);
  const int nst = (N + SS_NS - 1) / SS_NS;
  const int i0 = (DFM_BY % nst) * SS_NS, d0 = (DFM_BY / nst) * SIM_PD, t0 = DFM_BX * SS_TP;
  const int ni = (N - i0 < SS_NS) ? N - i0 : SS_NS, nt = (T - t0 < SS_TP) ? T - t0 : SS_TP;
  const int dn = (nb - d0 < SIM_PD) ? nb - d0 : SIM_PD;
  const int ld = em_lds(r), ldv = SS_TP + 1;
  double* Ls = sm;                                     // [SS_NS][ld]   loadings of the tile's series
  double* Fsh = Ls + (size_t)SS_NS * ld;               // [SS_TP][ld]   one replicate's factors of the tile's periods
  double* Cs = Fsh + (size_t)SS_TP * ld;               // [SS_NS][ldv]  lam_i' f_t
  double* Sd = Cs + (size_t)SS_NS * ldv;               // [SS_NS]       sqrt(R_i), NaN for a series out of the model
  unsigned char* obs = (unsigned char*)(Sd + SS_NS);   // [SS_NS][SS_TP] does the template observe the cell?
  for (int e = DFM_TID; e < SS_NS * r; e += DFM_NT) {
    const int i = e % SS_NS, a = e / SS_NS;
    Ls[i * ld + a] = (i < ni) ? Lam[i0 + i + (size_t)N * a] : 0.0;
  }
  for (int i = DFM_TID; i < SS_NS; i += DFM_NT) {
    bool in = i < ni && !is_nan(R[i0 + i]);
    for (int a = 0; a < r && in; ++a) if (is_nan(Lam[i0 + i + (size_t)N * a])) in = false;
    Sd[i] = in ? sqrt(R[i0 + i]) : DFM_NAN;
  }
  for (int e = DFM_TID; e < ni * SS_TP; e += DFM_NT) {
    const int i = e / SS_TP, t = e - i * SS_TP;
    obs[e] = (t < nt) ? !is_nan(Xt[(size_t)(i0 + i) * T + t0 + t]) : 0;
  }
  for (int d = 0; d < dn; ++d) {
    const int j = d0 + d;
    const unsigned long long id = (unsigned long long)(rep0 + j);
    DFM_SYNC();
    for (int e = DFM_TID; e < nt * r; e += DFM_NT) { const int t = e / r, a = e - t * r; Fsh[t * ld + a] = fS[((size_t)j * T + t0 + t) * r + a]; }
    DFM_SYNC();
    wt_gemm(Fsh, ld, 1, Ls, ld, 1, nt, ni, r, [&](int t, int i, double v) { Cs[i * ldv + t] = v; });
    DFM_SYNC();
    double* xo = Xout + (size_t)j * T * N;
    for (int e = DFM_TID; e < ni * SS_TP; e += DFM_NT) {
      const int i = e / SS_TP, t = e - i * SS_TP;
      if (t >= nt) continue;
      const double sd = Sd[i];
      double v = DFM_NAN;
      if (obs[e] && !is_nan(sd)) v = Cs[i * ldv + t] + sd * rng_normal(seed, id, RNG_SSB_EPS, (unsigned long long)(i0 + i) * T + t0 + t);
      xo[(size_t)(i0 + i) * T + t0 + t] = v;
    }
  }
}

// B copies of n doubles: dst[b n + e] = src[e].  grid-stride, grid.y = replicates.
__global__ void k_ss_bcast(const double* __restrict__ src, long long n, double* __restrict__ dst) {
  double* d = dst + (size_t)DFM_BY * n;
  for (long long e = (long long)DFM_BX * DFM_NT + DFM_TID; e < n; e += (long long)DFM_GX * DFM_NT) d[e] = src[e];
}

__host__ __device__ inline size_t ssb_align_smem_doubles(int r, int p) {
  const int k = r * p, ld = em_lds(r), ld2 = em_lds(2 * r);
  return (size_t)SSB_NC * ld + (size_t)SSB_NC * ld2 + 2 * (size_t)r * r + 2 * (size_t)r * 2 * r + 2 * (size_t)r * k + (size_t)r * ld + 2 * r + 8;
}

// Alignment of replicate b = DFM_BX (SSB_NT threads).  The EM estimates (Lam*, R*, A*, Q*) are identified up to f -> K f; with
// W = diag(1 / R^_i) over the series in the fitted model (Lam^ row and R^_i not NaN),
//   X = (Lam*' W Lam*)^-1 Lam*' W Lam^,  K = X^-1,  Lam~ = Lam* X,  A~_l = K A*_l X,  Q~ = K Q* K',  R~ = R*,
// the rotation that brings Lam* closest to Lam^ in the W-weighted least-squares sense (X = Lam^ exactly when Lam* = Lam^ K^-1).
// The N x r contractions and Lam* X are DMMA tile products over chunks of SSB_NC series.  Pivot rules (SSB_SING_TOL):
//   Lam*' W Lam*  singular when a Cholesky pivot <= tol * its largest diagonal entry (or is not > 0);
//   X             singular when a partial-pivoting Gauss-Jordan pivot |u_jj| <= tol * max |X_ij|;
//   Q~            not positive definite when a Cholesky pivot is not > 0.
// status[b] = the EM status when it is not 0, 3 when the alignment fails, else 0.  A failed replicate has NaN in Lo / Ao / Qo /
// Ro and in M / G (so its impulse responses are NaN); the E-step parameters Le / Re / Ae / Qe (may be NULL) then hold the fitted
// ones, so that a later E-step over the batch stays well defined.  llf[b] = the log-likelihood of the last EM iteration.
struct SsbAlignArgs {
  const double *Lh, *Rh, *Ah, *Qh;                     // fitted parameters (one model)
  const double *Ls, *Rs, *As, *Qs, *ll;                // EM results per replicate; ll [B][max_iter]
  const int *it, *em_status;
  double *Lo, *Ro, *Ao, *Qo;                           // aligned parameters (NaN for failed replicates)
  double *Le, *Re, *Ae, *Qe;                           // E-step parameters (may be NULL)
  double *M, *Qsel, *G;                                // companion form for dfm_irf: k x k, r x k, k x r
  double* llf; int* status;
  int N, r, p, max_iter;
};
__global__ void k_ss_align(SsbAlignArgs a) {
  DFM_SMEM(sm);
  const int b = DFM_BX, N = a.N, r = a.r, k = r * a.p, rr = r * r, rk = r * k;
  const int ld = em_lds(r), ld2 = em_lds(2 * r);
  double* S1 = sm;                                     // [SSB_NC][ld]   w_i lam*_i
  double* S2 = S1 + (size_t)SSB_NC * ld;               // [SSB_NC][ld2]  [lam*_i | lam^_i]
  double* Gm = S2 + (size_t)SSB_NC * ld2;              // r x r          Lam*' W Lam*, then its Cholesky factor
  double* Acc = Gm + rr;                               // r x 2r         [Lam*' W Lam* | Lam*' W Lam^]
  double* Aug = Acc + 2 * rr;                          // r x 2r         [X | I] -> [I | K]
  double* Xm = Aug + 2 * rr;                           // r x r          X
  double* T1 = Xm + rr;                                // r x k
  double* T2 = T1 + rk;                                // r x k
  double* Xt = T2 + rk;                                // [r][ld]        X' (the n operand of Lam* X)
  double* fac = Xt + (size_t)r * ld;                   // [r]            Gauss-Jordan column factors
  double* piv = fac + r;                               // [1]            the current pivot
  int* flag = (int*)(piv + r);                         // [0] failed  [1] pivot row  [2] Cholesky info
  const double* Ls = a.Ls + (size_t)b * N * r;
  const double* Rs = a.Rs + (size_t)b * N;
  if (DFM_TID == 0) { flag[0] = a.em_status[b] != 0; flag[2] = 0; }
  for (int e = DFM_TID; e < 2 * rr; e += DFM_NT) Acc[e] = 0.0;
  DFM_SYNC();
  // ---- Lam*' W [Lam* | Lam^] over chunks of series
  for (int c0 = 0; c0 < N; c0 += SSB_NC) {
    const int nc = (N - c0 < SSB_NC) ? N - c0 : SSB_NC;
    for (int i = DFM_TID; i < nc; i += DFM_NT) {
      const int g = c0 + i;
      bool in = !is_nan(a.Rh[g]);
      for (int c = 0; c < r && in; ++c) if (is_nan(a.Lh[g + (size_t)N * c])) in = false;
      const double w = in ? 1.0 / a.Rh[g] : 0.0;
      for (int c = 0; c < r; ++c) {
        const double ls = in ? Ls[g + (size_t)N * c] : 0.0;
        S1[i * ld + c] = w * ls;
        S2[i * ld2 + c] = ls;
        S2[i * ld2 + r + c] = in ? a.Lh[g + (size_t)N * c] : 0.0;
      }
    }
    DFM_SYNC();
    wt_gemm(S1, 1, ld, S2, 1, ld2, r, 2 * r, nc, [&](int m, int n, double v) { Acc[m + r * n] += v; });
    DFM_SYNC();
  }
  // ---- X = Gm^-1 Hm (Cholesky; relative pivot rule)
  double dmax = 0.0;
  for (int j = 0; j < r; ++j) dmax = fmax(dmax, Acc[j + r * j]);
  for (int e = DFM_TID; e < rr; e += DFM_NT) { Gm[e] = Acc[e]; Xm[e] = Acc[rr + e]; }
  DFM_SYNC();
  bm_chol(Gm, r, r, flag + 2);
  if (DFM_TID == 0) {
    bool bad = flag[2] != 0 || !(dmax > 0.0);
    for (int j = 0; j < r; ++j) if (!(Gm[j + r * j] * Gm[j + r * j] > SSB_SING_TOL * dmax)) bad = true;
    if (bad) flag[0] = 1;
  }
  DFM_SYNC();
  bm_trsm_lower(Gm, r, r, Xm, r, r);
  bm_trsm_lowerT(Gm, r, r, Xm, r, r);
  // ---- K = X^-1: Gauss-Jordan with partial pivoting on [X | I]
  double xmax = 0.0;
  for (int e = 0; e < rr; ++e) xmax = fmax(xmax, fabs(Xm[e]));
  for (int e = DFM_TID; e < 2 * rr; e += DFM_NT) { const int i = e % r, j = e / r; Aug[e] = (j < r) ? Xm[e] : ((i == j - r) ? 1.0 : 0.0); }
  DFM_SYNC();
  for (int j = 0; j < r; ++j) {
    if (DFM_TID == 0) {
      int pr = j; double pv = fabs(Aug[j + r * j]);
      for (int i = j + 1; i < r; ++i) if (fabs(Aug[i + r * j]) > pv) { pv = fabs(Aug[i + r * j]); pr = i; }
      if (!(pv > SSB_SING_TOL * xmax)) flag[0] = 1;
      flag[1] = pr;
    }
    DFM_SYNC();
    const int pr = flag[1];
    if (pr != j)
      for (int c = DFM_TID; c < 2 * r; c += DFM_NT) { const double t = Aug[j + r * c]; Aug[j + r * c] = Aug[pr + r * c]; Aug[pr + r * c] = t; }
    DFM_SYNC();
    if (DFM_TID == 0) piv[0] = Aug[j + r * j];
    DFM_SYNC();
    const double pinv = (piv[0] != 0.0) ? 1.0 / piv[0] : 0.0;
    for (int c = DFM_TID; c < 2 * r; c += DFM_NT) Aug[j + r * c] *= pinv;
    for (int i = DFM_TID; i < r; i += DFM_NT) fac[i] = (i == j) ? 0.0 : Aug[i + r * j];
    DFM_SYNC();
    for (int e = DFM_TID; e < 2 * rr; e += DFM_NT) { const int i = e % r, c = e / r; if (i != j) Aug[e] -= fac[i] * Aug[j + r * c]; }
    DFM_SYNC();
  }
  const double* Km = Aug + rr;                         // r x r
  // ---- A~_l = K A*_l X,  Q~ = K Q* K'
  const double* As = a.As + (size_t)b * rk;
  const double* Qs = a.Qs + (size_t)b * rr;
  bm_gemm(T1, r, Km, r, false, As, r, false, r, k, r, 1.0, 0.0);            // K [A*_1 .. A*_p]
  for (int l = 0; l < a.p; ++l)
    bm_gemm(T2 + (size_t)rr * l, r, T1 + (size_t)rr * l, r, false, Xm, r, false, r, r, r, 1.0, 0.0);
  bm_gemm(T1, r, Km, r, false, Qs, r, false, r, r, r, 1.0, 0.0);            // K Q*
  bm_gemm(Gm, r, T1, r, false, Km, r, true, r, r, r, 1.0, 0.0);             // K Q* K'
  bm_symmetrize(Gm, r, r);
  for (int e = DFM_TID; e < rr; e += DFM_NT) Acc[e] = Gm[e];                // (Q~ kept in Acc[0 .. rr))
  DFM_SYNC();
  if (DFM_TID == 0) flag[2] = 0;
  DFM_SYNC();
  bm_chol(Gm, r, r, flag + 2);                                              // L_Q~
  if (DFM_TID == 0 && flag[2]) flag[0] = 1;
  for (int e = DFM_TID; e < r * ld; e += DFM_NT) { const int c = e / ld, l = e - c * ld; Xt[e] = (l < r) ? Xm[l + r * c] : 0.0; }
  DFM_SYNC();
  const bool failed = flag[0] != 0;
  // ---- outputs
  double* Lo = a.Lo + (size_t)b * N * r;
  for (int c0 = 0; c0 < N; c0 += SSB_NC) {
    const int nc = (N - c0 < SSB_NC) ? N - c0 : SSB_NC;
    for (int e = DFM_TID; e < nc * r; e += DFM_NT) { const int i = e / r, c = e - i * r; S1[i * ld + c] = Ls[c0 + i + (size_t)N * c]; }
    DFM_SYNC();
    wt_gemm(S1, ld, 1, Xt, ld, 1, nc, r, r, [&](int i, int c, double v) { Lo[c0 + i + (size_t)N * c] = failed ? DFM_NAN : v; });
    DFM_SYNC();
  }
  for (int i = DFM_TID; i < N; i += DFM_NT) a.Ro[(size_t)b * N + i] = failed ? DFM_NAN : Rs[i];
  for (int e = DFM_TID; e < rk; e += DFM_NT) a.Ao[(size_t)b * rk + e] = failed ? DFM_NAN : T2[e];
  for (int e = DFM_TID; e < rr; e += DFM_NT) a.Qo[(size_t)b * rr + e] = failed ? DFM_NAN : Acc[e];
  if (a.Le) {
    for (int e = DFM_TID; e < N * r; e += DFM_NT) a.Le[(size_t)b * N * r + e] = failed ? a.Lh[e] : Lo[e];
    for (int i = DFM_TID; i < N; i += DFM_NT) a.Re[(size_t)b * N + i] = failed ? a.Rh[i] : Rs[i];
    for (int e = DFM_TID; e < rk; e += DFM_NT) a.Ae[(size_t)b * rk + e] = failed ? a.Ah[e] : T2[e];
    for (int e = DFM_TID; e < rr; e += DFM_NT) a.Qe[(size_t)b * rr + e] = failed ? a.Qh[e] : Acc[e];
  }
  for (int e = DFM_TID; e < k * k; e += DFM_NT) {
    const int i = e % k, j = e / k;
    a.M[(size_t)b * k * k + e] = failed ? DFM_NAN : (i < r) ? T2[i + r * j] : ((j == i - r) ? 1.0 : 0.0);
  }
  for (int e = DFM_TID; e < rk; e += DFM_NT) { const int i = e % r, j = e / r; a.Qsel[(size_t)b * rk + e] = (i == j) ? 1.0 : 0.0; }
  for (int e = DFM_TID; e < k * r; e += DFM_NT) {
    const int i = e % k, j = e / k;
    a.G[(size_t)b * k * r + e] = failed ? DFM_NAN : (i < r) ? Gm[i + r * j] : 0.0;
  }
  if (DFM_TID == 0) {
    const int it = a.it[b];
    a.llf[b] = (it > 0) ? a.ll[(size_t)b * a.max_iter + it - 1] : DFM_NAN;
    a.status[b] = a.em_status[b] != 0 ? a.em_status[b] : (failed ? 3 : 0);
  }
}

// The last `rows` periods of xhat / xvar ((Tp x N) per replicate) -> rows x N per replicate; NaN for a failed replicate.
// grid-stride over nb * N * rows elements.
__global__ void k_ss_fc_rows(const double* __restrict__ xh, const double* __restrict__ xv, int Tp, int N, int rows, int nb,
                             const int* __restrict__ status, double* __restrict__ oxh, double* __restrict__ oxv) {
  const long long n = (long long)nb * N * rows;
  for (long long e = (long long)DFM_BX * DFM_NT + DFM_TID; e < n; e += (long long)DFM_GX * DFM_NT) {
    const long long c = e / rows;                      // column (replicate b, series i)
    const int t = (int)(e - c * rows);
    const int b = (int)(c / N);
    const bool bad = status[b] != 0;
    const size_t src = (size_t)c * Tp + Tp - rows + t;
    if (oxh) oxh[e] = bad ? DFM_NAN : xh[src];
    if (oxv) oxv[e] = bad ? DFM_NAN : xv[src];
  }
}

}  // namespace dfm
