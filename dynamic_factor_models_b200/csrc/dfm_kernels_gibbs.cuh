// dfm_kernels_gibbs.cuh -- Gibbs sampler of the state-space DFM (dfm_gibbs): many chains as one batch.  The spec is
// tests/gibbs_oracle.py.  A sweep over a sub-batch of C chains is
//   ss_estep (the fixed-parameter E-step of dfm_kalman_smooth, one panel copy per chain at that chain's parameters)
//   k_sim_gains    the simulation smoother's gain table, one per chain (grid.y = chain)
//   k_gibbs_paths  the factor step: one warp per chain runs the simulation smoother's forward filter and backward smoother
//                  as warp mat-vecs, every period's gains read from L2 (G_t is k x (k + 2r), H_t k x 2k), with the normals of
//                  k_sim_paths
//   k_gibbs_stats  s_i = sum_{t obs} x_it f~_t for every series and chain: X' [F~_1 .. F~_C] (N x T by T x C r) as DMMA tile
//                  products, the panel tile shared by all the chains of a CTA
//   k_gibbs_draw   one CTA per chain: the Gram matrices of the path, the per-series conjugate draws of (lam_i, R_i) (S_i by the
//                  downdate S_all - sum_{t missing} f~_t f~_t'), the matrix-normal / inverse-Wishart draw of (A, Q); writes theta
//                  in place for the next sweep's E-step
// and, on kept sweeps, k_sim_project (pstride = 1) for the panel draws, k_ss_align + k_irf for the impulse responses.
// Random numbers: rng_normal / rng_uniform (dfm_kernels_rep.cuh) with replication id gibbs_id(c, s) = c 2^24 + s; the factor
// step uses the simulation smoother's tags 7-10, the parameter step
//   RNG_GB_NU   14  nu_i (lam_i = m_i + sqrt(R_i) L_i^-T nu_i)   element i r + a
//   RNG_GB_W    15  Bartlett B_ij (i > j), then Xi (k x r)       element i + r j;  r^2 + a + k b
//   RNG_GB_GN   16  normals of the Gamma sampler                 element 64 e + j (attempt j of Gamma number e)
//   RNG_GB_GU   17  uniforms of the Gamma sampler                element 64 e + j
// Gamma numbers: e = i for R_i (series i < N), e = N + j for the Bartlett diagonal j < r.
// dfm_gibbs_constrained (k_gibbs_draw_constr): a series with restriction rows H_i lam_i = h_i draws from the exact conditional
// under the prior N(0, R_i / kap_lam I) conditioned on the rows, with the same random numbers (tag 14 elements i r + a, Gamma
// number i):  lam*_i = the EM's correction of m_i (S~ = kap_lam I + S_i in place of S), h0 = H_i' (H_i H_i')^-1 h_i,
//   R_i = (b_R + (q_i - 2 s_i' lam*_i + lam*_i' S~ lam*_i - kap_lam |h0|^2) / 2) / Gamma(a_R + n_i / 2),
//   lam_i = the EM's correction of the unrestricted draw m_i + sqrt(R_i) L_i^-T nu_i.
#pragma once
#include "dfm_common.cuh"
#include "dfm_kernels_em.cuh"
#include "dfm_kernels_rep.cuh"
#include "dfm_kernels_sim.cuh"

namespace dfm {

enum { RNG_GB_NU = 14, RNG_GB_W = 15, RNG_GB_GN = 16, RNG_GB_GU = 17 };

#define GB_TRIES 64            // Marsaglia-Tsang attempts per Gamma number
#define GB_PW 4                // chains (warps) per CTA of k_gibbs_paths
#define GB_NS 32               // series per CTA of k_gibbs_stats
#define GB_NC 32               // factor columns (chain, factor) per CTA of k_gibbs_stats
#define GB_TT 32               // periods per step of k_gibbs_stats
#define GB_NT 128              // threads of k_gibbs_draw

struct GbPrior { double kap_lam, a_R, b_R, kap_A, nu_Q, s_Q; };

// Gamma(alpha, 1), alpha >= 1, Marsaglia & Tsang (2000), Gamma number e of id: attempt j reads element GB_TRIES e + j of the two
// streams.  After GB_TRIES rejections (probability < 1e-80 for alpha >= 1) the value is d = alpha - 1/3.
__device__ inline double gb_gamma(double alpha, unsigned long long seed, unsigned long long id, unsigned long long e) {
  const double d = alpha - 1.0 / 3.0, c = 1.0 / sqrt(9.0 * d);
  for (int j = 0; j < GB_TRIES; ++j) {
    const unsigned long long el = e * GB_TRIES + j;
    const double x = rng_normal(seed, id, RNG_GB_GN, el);
    const double t = 1.0 + c * x, v = t * t * t;
    if (!(v > 0.0)) continue;
    const double u = rng_uniform(seed, id, RNG_GB_GU, el);
    if (u < 1.0 - 0.0331 * (x * x) * (x * x) || log(u) < 0.5 * x * x + d * (1.0 - v + log(v))) return d * v;
  }
  return d;
}

// Once per call, per series (in-sample rows t < T of the padded panel X, Tp x N): n_i, q_i = sum x_it^2 and the list of the
// missing in-sample periods (midx[i T ..], mcnt[i]).  grid ceil(N / 128), 128 threads.
__global__ void k_gibbs_scan(const double* __restrict__ X, int T, int Tp, int N, int* __restrict__ nobs, double* __restrict__ q,
                             int* __restrict__ mcnt, int* __restrict__ midx) {
  for (int i = DFM_BX * DFM_NT + DFM_TID; i < N; i += DFM_GX * DFM_NT) {
    int n = 0, m = 0; double s = 0.0;
    for (int t = 0; t < T; ++t) {
      const double x = X[(size_t)i * Tp + t];
      if (is_nan(x)) midx[(size_t)i * T + m++] = t;
      else { ++n; s += x * x; }
    }
    nobs[i] = n; q[i] = s; mcnt[i] = m;
  }
}

__host__ __device__ inline size_t gibbs_paths_smem_doubles(int r, int p) {
  const size_t k = (size_t)r * p;
  return GB_PW * (6 * k + 3 * (size_t)r);
}

// The factor step of C chains: chain c = DFM_BX * GB_PW + w runs on warp w.  Per chain: gains (sim_gains_doubles apart, from
// k_sim_gains), cst[c] (the chain's status; != 0: NaN F, zero fS).  The forward and backward recursions of k_sim_paths with the
// same normals (tags 7-9, id = id0 + c idstride); each lane owns rows lane, lane + 32 of the k x (k + 2r) and k x 2k mat-vecs.
// Writes fS [Tp][C][r] (f~_t), z0 [C][k] (z~_0: its lag block supplies the pre-sample lags of the transition step), zf scratch
// [C][Tp][k], and Fout (Tp x r column-major per chain; may be NULL).
__global__ void k_gibbs_paths(const double* __restrict__ gains, int Tp, int r, int p, int C,
                              unsigned long long seed, long long id0, long long idstride, const int* __restrict__ cst,
                              double* __restrict__ zfS, double* __restrict__ fS, double* __restrict__ z0, double* __restrict__ Fout) {
  DFM_SMEM(sm);
  const int k = r * p, kk = k * k, kr2 = k + 2 * r;
  const size_t gstr = sim_gain_stride(k, r), gall = sim_gains_doubles(Tp, k, r);
  for (int w = DFM_WARP; w < GB_PW; w += DFM_NWARP) {
    const int c = DFM_BX * GB_PW + w;
    if (c >= C) continue;
    double* P = sm + (size_t)w * (6 * k + 3 * r);    // [z+ | eta]     k + r
    double* Wv = P + k + r;                            // [zf | f+ | xi] k + 2r
    double* Yv = Wv + kr2;                             // [zf_t | zs_t+1] 2k
    double* z0p = Yv + 2 * k;                          // z+_0           k
    double* tmp = z0p + k;                             //                k
    const int lane = DFM_LANE;
    double* zf = zfS + (size_t)c * Tp * k;
    if (cst[c] != 0) {
      for (int e = lane; e < Tp * r; e += DFM_WSZ) {
        const int t = e / r, a = e - t * r;
        fS[((size_t)t * C + c) * r + a] = 0.0;
        if (Fout) Fout[(size_t)c * Tp * r + t + (size_t)Tp * a] = DFM_NAN;
      }
      for (int i = lane; i < k; i += DFM_WSZ) z0[(size_t)c * k + i] = 0.0;
      continue;
    }
    const double* gc = gains + (size_t)c * gall;
    const double* LP0 = gc + (size_t)Tp * gstr;
    const double* AQ = LP0 + kk;                       // [A | L_Q]  r x (k + r)
    const unsigned long long id = (unsigned long long)(id0 + (long long)c * idstride);
    for (int i = lane; i < k; i += DFM_WSZ) { P[i] = rng_normal(seed, id, RNG_SS_Z0, i); Wv[i] = 0.0; }
    DFM_WSYNC();
    for (int i = lane; i < k; i += DFM_WSZ) {
      double s = 0.0;
      for (int j = 0; j <= i; ++j) s += LP0[i + (size_t)k * j] * P[j];
      tmp[i] = s;
    }
    DFM_WSYNC();
    for (int i = lane; i < k; i += DFM_WSZ) { P[i] = tmp[i]; z0p[i] = tmp[i]; }
    DFM_WSYNC();
    // ---------------------------------------------------------------- forward
    for (int t = 0; t < Tp; ++t) {
      if (t > 0) {
        for (int a = lane; a < r; a += DFM_WSZ) P[k + a] = rng_normal(seed, id, RNG_SS_ETA, (unsigned long long)t * r + a);
        DFM_WSYNC();
        for (int i = lane; i < k; i += DFM_WSZ) {
          double s = 0.0;
          if (i < r) { for (int j = 0; j < k + r; ++j) s += AQ[i + (size_t)r * j] * P[j]; }
          else s = P[i - r];
          tmp[i] = s;
        }
        DFM_WSYNC();
        for (int i = lane; i < k; i += DFM_WSZ) P[i] = tmp[i];
      }
      for (int a = lane; a < r; a += DFM_WSZ) Wv[k + r + a] = rng_normal(seed, id, RNG_SS_OBS, (unsigned long long)t * r + a);
      DFM_WSYNC();
      for (int a = lane; a < r; a += DFM_WSZ) { Wv[k + a] = P[a]; fS[((size_t)t * C + c) * r + a] = P[a]; }
      DFM_WSYNC();
      const double* G = gc + (size_t)t * gstr;
      const double* kb = G + (size_t)k * kr2;
      for (int i = lane; i < k; i += DFM_WSZ) {
        double s0 = 0.0, s1 = 0.0;
        int j = 0;
        for (; j + 1 < kr2; j += 2) { s0 += G[i + (size_t)k * j] * Wv[j]; s1 += G[i + (size_t)k * (j + 1)] * Wv[j + 1]; }
        if (j < kr2) s0 += G[i + (size_t)k * j] * Wv[j];
        tmp[i] = (s0 + s1) + kb[i];
      }
      DFM_WSYNC();
      for (int i = lane; i < k; i += DFM_WSZ) { Wv[i] = tmp[i]; zf[(size_t)t * k + i] = tmp[i]; }
      DFM_WSYNC();
    }
    // ---------------------------------------------------------------- backward
    for (int i = lane; i < k; i += DFM_WSZ) Yv[k + i] = Wv[i];
    for (int a = lane; a < r; a += DFM_WSZ) {
      const size_t o = ((size_t)(Tp - 1) * C + c) * r + a;
      const double f = fS[o] + Wv[a];
      fS[o] = f;
      if (Fout) Fout[(size_t)c * Tp * r + (Tp - 1) + (size_t)Tp * a] = f;
    }
    DFM_WSYNC();
    for (int t = Tp - 2; t >= 0; --t) {
      for (int i = lane; i < k; i += DFM_WSZ) Yv[i] = zf[(size_t)t * k + i];
      DFM_WSYNC();
      const double* Hm = gc + (size_t)t * gstr + (size_t)k * kr2 + k;
      for (int i = lane; i < k; i += DFM_WSZ) {
        double s0 = 0.0, s1 = 0.0;
        for (int j = 0; j < 2 * k; j += 2) { s0 += Hm[i + (size_t)k * j] * Yv[j]; s1 += Hm[i + (size_t)k * (j + 1)] * Yv[j + 1]; }
        tmp[i] = s0 + s1;
      }
      DFM_WSYNC();
      for (int i = lane; i < k; i += DFM_WSZ) Yv[k + i] = tmp[i];
      for (int a = lane; a < r; a += DFM_WSZ) {
        const size_t o = ((size_t)t * C + c) * r + a;
        const double f = fS[o] + tmp[a];
        fS[o] = f;
        if (Fout) Fout[(size_t)c * Tp * r + t + (size_t)Tp * a] = f;
      }
      DFM_WSYNC();
    }
    for (int i = lane; i < k; i += DFM_WSZ) z0[(size_t)c * k + i] = z0p[i] + Yv[k + i];
    DFM_WSYNC();
  }
}

__host__ __device__ inline size_t gibbs_stats_smem_doubles() {
  const int ld = em_lds(GB_TT);
  return (size_t)GB_NS * ld + (size_t)GB_NC * ld + (size_t)GB_NS * GB_NC;
}

// s_i for every series and chain: sv[c][i + N a] = sum_{t < T, x_it observed} x_it f~_t,a, i.e. X' [F~_1 .. F~_C] with the
// missing cells as 0.  X: padded panel (Tp x N, the first copy); fS [Tp][C][r] (column j = c r + a of F~ is contiguous in j).
// CTA (series tile of GB_NS, column tile of GB_NC): the panel tile and the factor tile of GB_TT periods staged in shared memory,
// DMMA tile products accumulated in shared memory.  grid (ceil(N / GB_NS), ceil(C r / GB_NC)), 128 threads.
__global__ void k_gibbs_stats(const double* __restrict__ X, const double* __restrict__ fS, int T, int Tp, int N, int r, int C,
                              double* __restrict__ sv) {
  DFM_SMEM(sm);
  const int ld = em_lds(GB_TT);
  const int i0 = DFM_BX * GB_NS, j0 = DFM_BY * GB_NC, Cr = C * r;
  const int ni = (N - i0 < GB_NS) ? N - i0 : GB_NS, nj = (Cr - j0 < GB_NC) ? Cr - j0 : GB_NC;
  double* Xs = sm;                                     // [GB_NS][ld]
  double* Fs = Xs + (size_t)GB_NS * ld;                // [GB_NC][ld]
  double* Acc = Fs + (size_t)GB_NC * ld;               // [GB_NC][GB_NS]
  for (int e = DFM_TID; e < GB_NS * GB_NC; e += DFM_NT) Acc[e] = 0.0;
  for (int t0 = 0; t0 < T; t0 += GB_TT) {
    const int nt = (T - t0 < GB_TT) ? T - t0 : GB_TT;
    for (int e = DFM_TID; e < GB_NS * GB_TT; e += DFM_NT) {
      const int i = e / GB_TT, t = e - i * GB_TT;
      double x = 0.0;
      if (i < ni && t < nt) { x = X[(size_t)(i0 + i) * Tp + t0 + t]; if (is_nan(x)) x = 0.0; }
      Xs[i * ld + t] = x;
    }
    for (int e = DFM_TID; e < GB_NC * GB_TT; e += DFM_NT) {
      const int t = e / GB_NC, j = e - t * GB_NC;
      Fs[j * ld + t] = (j < nj && t < nt) ? fS[(size_t)(t0 + t) * Cr + j0 + j] : 0.0;
    }
    DFM_SYNC();
    wt_gemm(Xs, ld, 1, Fs, ld, 1, ni, nj, nt, [&](int i, int j, double v) { Acc[j * GB_NS + i] += v; });
    DFM_SYNC();
  }
  for (int e = DFM_TID; e < ni * nj; e += DFM_NT) {
    const int j = e / ni, i = e - j * ni;
    const int col = j0 + j, c = col / r, a = col - c * r;
    sv[(size_t)c * N * r + i0 + i + (size_t)N * a] = Acc[j * GB_NS + i];
  }
}

__host__ __device__ inline size_t gibbs_draw_smem_doubles(int r, int p) {
  const size_t k = (size_t)r * p;
  return 3 * k * k + 4 * k * r + 7 * (size_t)r * r + 2 * k + 8;
}

// Per-chain scratch of k_gibbs_draw's series phase: (r (r + 1) / 2 + 2 r) x N doubles, element (e, i) at e N + i.
__host__ __device__ inline size_t gibbs_draw_wk_doubles(int N, int r) { return ((size_t)r * (r + 1) / 2 + 2 * (size_t)r) * N; }

struct GibbsDrawArgs {
  const double *X, *fS, *z0, *sv, *q;                  // padded panel (first copy), paths, z~_0, s_i, q_i
  const int *nobs, *mcnt, *midx;
  double *Lam, *R, *A, *Q;                             // theta of every chain, updated in place
  double* wk;                                          // [C] gibbs_draw_wk_doubles
  int* cst;                                            // chain status
  GbPrior pr;
  int T, Tp, N, r, p, C;
  unsigned long long seed; long long id0, idstride;
};

// Shared scratch of k_gibbs_draw_constr's restricted pass (doubles, after gibbs_draw_smem_doubles): lam_constr_correct's
// scratch, then three r-vectors.
__host__ __device__ inline size_t gibbs_constr_smem_doubles(int r) { return (size_t)em_constr_scratch(r) + 3 * (size_t)r; }

// One CTA per chain (GB_NT threads): the parameter step of the sweep at the path of k_gibbs_paths (steps 2-3 of the spec).
// A chain whose status is not 0 keeps its parameters; a Cholesky factor that is not positive definite sets status 3.
// CON (k_gibbs_draw_constr, the call has restriction rows cs): the thread-per-series loop leaves the restricted series after
// their Cholesky solve (L_i and m_i stay in wk); thread 0 then draws them one by one (header comment), with the scratch of
// gibbs_constr_smem_doubles in shared memory.  Dependent rows set status 3.  Without CON the body is the unrestricted kernel.
template <bool CON>
__device__ __forceinline__ void gibbs_draw_body(GibbsDrawArgs a, EmConstr cs) {
  DFM_SMEM(sm);
  const int c = DFM_BX, r = a.r, p = a.p, k = r * p, T = a.T, N = a.N, C = a.C, kk = k * k, rr = r * r, rk = r * k;
  const int np = r * (r + 1) / 2;
  if (a.cst[c] != 0) return;
  const unsigned long long id = (unsigned long long)(a.id0 + (long long)c * a.idstride);
  double* ZZ = sm;           double* LZ = ZZ + kk;      double* T3 = LZ + kk;
  double* ZY = T3 + kk;      double* Bh = ZY + rk;      double* Xi = Bh + rk;      double* At = Xi + rk;
  double* Sa = At + rk;      double* YY = Sa + rr;      double* S = YY + rr;       double* Bm = S + rr;
  double* Ut = Bm + rr;      double* Qn = Ut + rr;      double* LQ = Qn + rr;
  double* zc = LQ + rr;      // [2k] z~_0 of the chain, pre-sample lags
  int* info = (int*)(zc + 2 * k);
  const double* fS = a.fS;
  const double* z0 = a.z0 + (size_t)c * k;
  // f_ext(u, b): f~_u for u >= 0, the lag block of z~_0 for u < 0
  auto fx = [&](int u, int b) -> double { return u >= 0 ? fS[((size_t)u * C + c) * r + b] : zc[(-u) * r + b]; };
  for (int i = DFM_TID; i < k; i += DFM_NT) zc[i] = z0[i];
  if (DFM_TID == 0) { info[0] = 0; info[1] = 0; }
  DFM_SYNC();
  // ---- Gram matrices: S_all (t < T), Z'Z, Z'Y, Y'Y (t = 1 .. T-1; Z_t[b + r l] = f_ext(t - 1 - l, b))
  for (int e = DFM_TID; e < rr; e += DFM_NT) {
    const int x = e % r, y = e / r;
    double s = 0.0, s2 = 0.0;
    for (int t = 0; t < T; ++t) { const double v = fx(t, x) * fx(t, y); s += v; if (t > 0) s2 += v; }
    Sa[e] = s; YY[e] = s2;
  }
  for (int e = DFM_TID; e < kk; e += DFM_NT) {
    const int x = e % k, y = e / k, bx = x % r, lx = x / r, by = y % r, ly = y / r;
    double s = 0.0;
    for (int t = 1; t < T; ++t) s += fx(t - 1 - lx, bx) * fx(t - 1 - ly, by);
    ZZ[e] = s;
  }
  for (int e = DFM_TID; e < rk; e += DFM_NT) {
    const int x = e % k, y = e / k, bx = x % r, lx = x / r;
    double s = 0.0;
    for (int t = 1; t < T; ++t) s += fx(t - 1 - lx, bx) * fx(t, y);
    ZY[e] = s;
  }
  DFM_SYNC();
  // ---- measurement step: one thread per series
  double* Lam = a.Lam + (size_t)c * N * r;
  double* Rv = a.R + (size_t)c * N;
  double* wk = a.wk + (size_t)c * gibbs_draw_wk_doubles(N, r);
  const double* sv = a.sv + (size_t)c * N * r;
  for (int i = DFM_TID; i < N; i += DFM_NT) {
    bool in = !is_nan(Rv[i]);
    for (int b = 0; b < r && in; ++b) if (is_nan(Lam[i + (size_t)N * b])) in = false;
    if (!in) continue;
    double* Ap = wk + i;                               // packed kap I + S_i, stride N
    double* bv = wk + (size_t)np * N + i;              // s_i -> m_i
    double* s0 = wk + (size_t)(np + r) * N + i;        // s_i
    for (int x = 0; x < r; ++x)
      for (int y = 0; y <= x; ++y) {
        double v = Sa[x + r * y] + (x == y ? a.pr.kap_lam : 0.0);
        const int nm = a.mcnt[i];
        for (int m = 0; m < nm; ++m) { const int t = a.midx[(size_t)i * T + m]; v -= fx(t, x) * fx(t, y); }
        Ap[(size_t)pidx(x, y) * N] = v;
      }
    for (int x = 0; x < r; ++x) { const double v = sv[i + (size_t)N * x]; bv[(size_t)x * N] = v; s0[(size_t)x * N] = v; }
    if (chol_solve_packed(Ap, bv, r, N)) { atomicMax(&info[1], 1); continue; }
    if constexpr (CON) { if (cs.off[i + 1] > cs.off[i]) continue; }     // restricted: drawn below
    double sm_ = 0.0;
    for (int x = 0; x < r; ++x) sm_ += s0[(size_t)x * N] * bv[(size_t)x * N];
    const double al = a.pr.a_R + 0.5 * a.nobs[i], be = a.pr.b_R + 0.5 * (a.q[i] - sm_);
    const double Ri = be / gb_gamma(al, a.seed, id, (unsigned long long)i);
    const double sr = sqrt(Ri);
    // L_i^-T nu_i into s0 (back substitution with the packed factor)
    for (int x = r - 1; x >= 0; --x) {
      double s = rng_normal(a.seed, id, RNG_GB_NU, (unsigned long long)i * r + x);
      for (int y = x + 1; y < r; ++y) s -= Ap[(size_t)pidx(y, x) * N] * s0[(size_t)y * N];
      s0[(size_t)x * N] = s / Ap[(size_t)pidx(x, x) * N];
    }
    Rv[i] = Ri;
    for (int x = 0; x < r; ++x) Lam[i + (size_t)N * x] = bv[(size_t)x * N] + sr * s0[(size_t)x * N];
  }
  if constexpr (CON) {
    DFM_SYNC();
    if (DFM_TID == 0) {
      double* ws = zc + 2 * k + 8;                     // (info occupies the 8 doubles after zc)
      double* lv = ws + em_constr_scratch(r);          // lam*, then the draw
      double* h0 = lv + r;                             // H_i' (H_i H_i')^-1 h_i
      double* uv = h0 + r;
      for (int i = 0; i < N && !info[1]; ++i) {
        const int q0 = cs.off[i], m = cs.off[i + 1] - q0;
        bool in = m > 0 && !is_nan(Rv[i]);
        for (int b = 0; b < r && in; ++b) if (is_nan(Lam[i + (size_t)N * b])) in = false;
        if (!in) continue;
        const double* Ap = wk + i;                     // L_i (packed, stride N)
        const double* bv = wk + (size_t)np * N + i;    // m_i
        const double* s0 = wk + (size_t)(np + r) * N + i;
        const double* Hq = cs.H + (size_t)q0 * r;
        const double* hq = cs.h + q0;
        auto solve = [&](double* v) {                  // v <- S~^-1 v
          for (int x = 0; x < r; ++x) {
            double s = v[x];
            for (int y = 0; y < x; ++y) s -= Ap[(size_t)pidx(x, y) * N] * v[y];
            v[x] = s / Ap[(size_t)pidx(x, x) * N];
          }
          for (int x = r - 1; x >= 0; --x) {
            double s = v[x];
            for (int y = x + 1; y < r; ++y) s -= Ap[(size_t)pidx(y, x) * N] * v[y];
            v[x] = s / Ap[(size_t)pidx(x, x) * N];
          }
        };
        for (int x = 0; x < r; ++x) { h0[x] = 0.0; lv[x] = bv[(size_t)x * N]; }
        if (lam_constr_correct(h0, r, Hq, hq, m, ws, [](double*) {}) || lam_constr_correct(lv, r, Hq, hq, m, ws, solve)) {
          info[1] = 1;
          break;
        }
        double sl = 0.0, q2 = 0.0, n0 = 0.0;
        for (int x = 0; x < r; ++x) {
          double v = 0.0;                              // (L_i' lam*)_x
          for (int y = x; y < r; ++y) v += Ap[(size_t)pidx(y, x) * N] * lv[y];
          q2 += v * v; sl += s0[(size_t)x * N] * lv[x]; n0 += h0[x] * h0[x];
        }
        const double al = a.pr.a_R + 0.5 * a.nobs[i];
        const double be = a.pr.b_R + 0.5 * (a.q[i] - 2.0 * sl + q2 - a.pr.kap_lam * n0);
        const double Ri = be / gb_gamma(al, a.seed, id, (unsigned long long)i);
        const double sr = sqrt(Ri);
        for (int x = r - 1; x >= 0; --x) {              // L_i^-T nu_i
          double s = rng_normal(a.seed, id, RNG_GB_NU, (unsigned long long)i * r + x);
          for (int y = x + 1; y < r; ++y) s -= Ap[(size_t)pidx(y, x) * N] * uv[y];
          uv[x] = s / Ap[(size_t)pidx(x, x) * N];
        }
        for (int x = 0; x < r; ++x) uv[x] = bv[(size_t)x * N] + sr * uv[x];
        if (lam_constr_correct(uv, r, Hq, hq, m, ws, solve)) { info[1] = 1; break; }
        Rv[i] = Ri;
        for (int x = 0; x < r; ++x) Lam[i + (size_t)N * x] = uv[x];
      }
    }
  }
  // ---- transition step
  for (int e = DFM_TID; e < kk; e += DFM_NT) { const int x = e % k, y = e / k; LZ[e] = ZZ[e] + (x == y ? a.pr.kap_A : 0.0); }
  for (int e = DFM_TID; e < rk; e += DFM_NT) Bh[e] = ZY[e];
  DFM_SYNC();
  bm_chol(LZ, k, k, info);
  bm_trsm_lower(LZ, k, k, Bh, k, r);
  bm_trsm_lowerT(LZ, k, k, Bh, k, r);                                        // B^ = (kap I + Z'Z)^-1 Z'Y
  for (int e = DFM_TID; e < rr; e += DFM_NT) { const int x = e % r, y = e / r; S[e] = YY[e] + (x == y ? a.pr.s_Q : 0.0); }
  DFM_SYNC();
  bm_gemm(S, r, Bh, k, true, ZY, k, false, r, r, k, -1.0, 1.0);             // S = s_Q I + Y'Y - B^' Z'Y
  bm_symmetrize(S, r, r);
  bm_chol(S, r, r, info);                                                    // L
  const double nu = a.pr.nu_Q + T - 1;
  for (int e = DFM_TID; e < rr; e += DFM_NT) {
    const int x = e % r, y = e / r;
    Bm[e] = (x > y) ? rng_normal(a.seed, id, RNG_GB_W, (unsigned long long)e) : 0.0;
    Ut[e] = S[y + r * x];                                                    // L'
  }
  for (int j = DFM_TID; j < r; j += DFM_NT)
    Bm[j + r * j] = sqrt(2.0 * gb_gamma(0.5 * (nu - j), a.seed, id, (unsigned long long)N + j));
  for (int e = DFM_TID; e < rk; e += DFM_NT) Xi[e] = rng_normal(a.seed, id, RNG_GB_W, (unsigned long long)rr + e);
  DFM_SYNC();
  bm_trsm_lower(Bm, r, r, Ut, r, r);                                         // U' = B^-1 L'
  bm_gemm(Qn, r, Ut, r, true, Ut, r, false, r, r, r, 1.0, 0.0);             // Q = U U'
  bm_symmetrize(Qn, r, r);
  for (int e = DFM_TID; e < rr; e += DFM_NT) LQ[e] = Qn[e];
  DFM_SYNC();
  bm_chol(LQ, r, r, info);
  bm_trsm_lowerT(LZ, k, k, Xi, k, r);                                        // L_Z^-T Xi
  for (int e = DFM_TID; e < rk; e += DFM_NT) At[e] = Bh[e];
  DFM_SYNC();
  bm_gemm(At, k, Xi, k, false, LQ, r, true, k, r, r, 1.0, 1.0);             // A' = B^ + L_Z^-T Xi L_Q'
  if (info[0] || info[1]) { if (DFM_TID == 0) a.cst[c] = 3; return; }
  double* Ao = a.A + (size_t)c * rk;
  double* Qo = a.Q + (size_t)c * rr;
  for (int e = DFM_TID; e < rk; e += DFM_NT) { const int x = e % r, y = e / r; Ao[e] = At[y + k * x]; }
  for (int e = DFM_TID; e < rr; e += DFM_NT) Qo[e] = Qn[e];
}

__global__ void k_gibbs_draw(GibbsDrawArgs a) { gibbs_draw_body<false>(a, EmConstr{nullptr, nullptr, nullptr}); }
__global__ void k_gibbs_draw_constr(GibbsDrawArgs a, EmConstr cs) { gibbs_draw_body<true>(a, cs); }

// dst[c * dstride + e] = src[c * sstride + e] for e < n, NaN where cst[c] != 0 (the records of a kept sweep).  grid (.., C).
__global__ void k_gibbs_rec(const double* __restrict__ src, long long sstride, long long n, const int* __restrict__ cst,
                            double* __restrict__ dst, long long dstride) {
  const int c = DFM_BY;
  const bool bad = cst[c] != 0;
  for (long long e = (long long)DFM_BX * DFM_NT + DFM_TID; e < n; e += (long long)DFM_GX * DFM_NT)
    dst[(size_t)c * dstride + e] = bad ? DFM_NAN : src[(size_t)c * sstride + e];
}

// out[c] = 3 if the chain failed, else 0.
__global__ void k_gibbs_status(const int* __restrict__ cst, int C, int* __restrict__ out) {
  for (int c = DFM_BX * DFM_NT + DFM_TID; c < C; c += DFM_GX * DFM_NT) out[c] = cst[c] != 0 ? 3 : 0;
}

}  // namespace dfm
