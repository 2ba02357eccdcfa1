// dfm_kernels_proxy.cuh -- shocks identified by external instruments (proxy SVAR / SVAR-IV) for many models at once
// (dfm_proxy_identification).  Per model (Lam, R, A, Q) and factor path f: L = chol(Q), eta_t = f_t - sum_l A_l f_{t-l},
// u_t = L^-1 eta_t; per instrument k over its periods T_k: g_k = (1/n_k) sum u_t (z_t - zbar) = L^-1 Gamma_k and the unit
// column omega_k = g_k / |g_k| (include/dfm_b200.h has the definition):
//   k_sr_prep, k_irf  (dfm_kernels_resp.cuh, dfm_kernels_np.cuh) L and Psi_h of every model
//   k_iv_prep         one CTA per model: u_t, and per instrument T_k, zbar, s^2, omega_k, eps_k, rho^2_k, the HAC first stage and
//                     the status
//   k_iv_boot         one thread per moving-block bootstrap replicate rho >= 1 of one (model, instrument): the model's compacted
//                     (u_t, z_t) in shared memory, the block starts from Philox tag 20, omega*
//   k_iv_rot          one CTA per record (model, instrument, replicate): Omega = the Householder completion of omega (first
//                     column omega), the records Psi_h Omega in k_irf's layout
//   k_series_resp     (dfm_kernels_resp.cuh) n_shock = 1 on those records
// Every sum runs in a fixed order in one thread, so the bits do not depend on the launch shape, the chunking or n_boot.  Plain FMA
// code: the host-emulation build runs the same source.  The spec is tests/proxy_oracle.py.
#pragma once
#include "dfm_common.cuh"
#include "dfm_kernels_rep.cuh"

namespace dfm {

enum { RNG_PROXY = 20 };       // block start j of replicate rho of instrument k: uniform number (rho n_inst + k) Tp + j

#define IV_PT 128              // threads of k_iv_prep
#define IV_BT 64               // replicates (threads) per CTA of k_iv_boot
#define IV_NIMAX 8             // instruments per call

// Shared memory of k_iv_prep: L (r r), y_t and h_t (2 Tp), g (r), 8 scalars, the row flags (Tp ints).
__host__ __device__ inline size_t iv_prep_smem_bytes(int r, int Tp) {
  return ((size_t)r * r + 2 * (size_t)Tp + r + 8) * 8 + (size_t)Tp * 4;
}

// grid (B), IV_PT threads.  A r x k, Lam N x r, R N per model; G: k_sr_prep's [L; 0] (k x r, NaN for a failed model); F: Tp x r per
// model; Z: Tp x ni (common to all models).  st[b]: k_sr_prep's status.  Writes U (u_t, Tp x r per model, NaN for t < p and rows
// with a NaN in f_t .. f_{t-p}), per (model, instrument) bk = b ni + k: idx (the n_k periods of T_k, ascending, Tp ints), nk, ist
// (status), om[bk (1 + n_boot) r ..] (omega, replicate 0), eps (Tp), nobs, rel, fpi, fF.
__global__ void k_iv_prep(const double* __restrict__ Lam, const double* __restrict__ R, const double* __restrict__ A,
                          const double* __restrict__ G, const double* __restrict__ F, const double* __restrict__ Z, int N, int r, int p,
                          int Tp, int ni, int i0, int q, int n_boot, const int* __restrict__ st, double* __restrict__ U,
                          int* __restrict__ idx, int* __restrict__ nk, int* __restrict__ ist, double* __restrict__ om,
                          double* __restrict__ eps, int* __restrict__ nobs, double* __restrict__ rel, double* __restrict__ fpi,
                          double* __restrict__ fF) {
  DFM_SMEM(sm);
  const int b = DFM_BX, k = r * p;
  double* sL = sm;                                     // [a + r c] L
  double* sY = sL + (size_t)r * r;                     // [t]  y_t = lam_i0' eta_t
  double* sH = sY + Tp;                                // [i]  the first stage's h_i
  double* sG = sH + Tp;                                // [a]  g, then omega
  double* red = sG + r;                                // [0] zbar [1] s^2 [2] status [3] n
  int* sBad = (int*)(red + 8);                         // [t]  1: a NaN in f_t .. f_{t-p} (or t < p)
  const double* Ab = A + (size_t)b * r * k;
  const double* Lb = Lam + (size_t)b * N * r;
  const double* Fb = F + (size_t)b * Tp * r;
  double* Ub = U + (size_t)b * Tp * r;
  for (int e = DFM_TID; e < r * r; e += DFM_NT) {
    const int a = e % r, c = e / r;
    sL[e] = a >= c ? G[(size_t)b * k * r + a + (size_t)k * c] : 0.0;
  }
  bool i0bad = is_nan(R[(size_t)b * N + i0]);
  for (int a = 0; a < r; ++a) i0bad = i0bad || is_nan(Lb[i0 + (size_t)N * a]);
  DFM_SYNC();
  for (int t = DFM_TID; t < Tp; t += DFM_NT) {
    bool bad = t < p;
    for (int l = 0; l <= p && !bad; ++l)
      for (int a = 0; a < r; ++a) bad = bad || is_nan(Fb[t - l + (size_t)Tp * a]);
    sBad[t] = bad ? 1 : 0;
    if (bad) {
      for (int a = 0; a < r; ++a) Ub[t + (size_t)Tp * a] = DFM_NAN;
      sY[t] = DFM_NAN;
      continue;
    }
    double y = 0.0;
    for (int a = 0; a < r; ++a) {                      // eta_{t,a}
      double e = Fb[t + (size_t)Tp * a];
      for (int l = 1; l <= p; ++l)
        for (int c = 0; c < r; ++c) e = fma(-Ab[a + (size_t)r * ((l - 1) * r + c)], Fb[t - l + (size_t)Tp * c], e);
      Ub[t + (size_t)Tp * a] = e;
      y = fma(Lb[i0 + (size_t)N * a], e, y);
    }
    sY[t] = y;
    for (int a = 0; a < r; ++a) {                      // u = L^-1 eta in place
      double s = Ub[t + (size_t)Tp * a];
      for (int c = 0; c < a; ++c) s = fma(-sL[a + r * c], Ub[t + (size_t)Tp * c], s);
      Ub[t + (size_t)Tp * a] = s / sL[a + r * a];
    }
  }
  DFM_SYNC();
  for (int kk = 0; kk < ni; ++kk) {
    const size_t bk = (size_t)b * ni + kk;
    const double* z = Z + (size_t)Tp * kk;
    int* ix = idx + bk * Tp;
    if (DFM_TID == 0) {
      int n = 0, pathbad = 0;
      for (int t = p; t < Tp; ++t)
        if (!is_nan(z[t])) { if (sBad[t]) pathbad = 1; else ix[n++] = t; }
      int code = st[b] != 0 ? 3 : (i0bad ? DFM_ERR_ARG : (pathbad || n < 3 ? 3 : 0));
      double zb = 0.0, s2 = 0.0;
      for (int i = 0; i < n; ++i) zb += z[ix[i]];
      zb /= (double)n;
      for (int i = 0; i < n; ++i) { const double d = z[ix[i]] - zb; s2 = fma(d, d, s2); }
      red[0] = zb; red[1] = s2 / (double)n; red[2] = (double)code; red[3] = (double)n;
    }
    DFM_SYNC();
    const int n = (int)red[3];
    const double zb = red[0];
    if ((int)red[2] == 0)
      for (int a = DFM_TID; a < r; a += DFM_NT) {
        double g = 0.0;
        for (int i = 0; i < n; ++i) g = fma(Ub[ix[i] + (size_t)Tp * a], z[ix[i]] - zb, g);
        sG[a] = g / (double)n;
      }
    DFM_SYNC();
    if (DFM_TID == 0) {
      int code = (int)red[2];
      double nrm2 = 0.0;
      if (code == 0) for (int a = 0; a < r; ++a) nrm2 = fma(sG[a], sG[a], nrm2);
      if (code == 0 && !(nrm2 > 0.0 && nrm2 < INFINITY)) code = 3;   // Gamma_k = 0
      double pi = DFM_NAN, Fs = DFM_NAN, rho2 = DFM_NAN;
      if (code == 0) {
        const double inv = 1.0 / sqrt(nrm2), s2 = red[1];
        for (int a = 0; a < r; ++a) sG[a] *= inv;
        rho2 = nrm2 / s2;
        // first stage: y_t on [1, z_t] over T_k; V = hac(v, X, q)[1, 1] = sum_{|j| <= q} w_j sum_i h_i h_{i+|j|} with
        // h_i = v_i (z_i - zbar) / sxx, the second row of (X'X)^-1 X_i' v_i
        double yb = 0.0, sxx = 0.0, sxy = 0.0;
        for (int i = 0; i < n; ++i) yb += sY[ix[i]];
        yb /= (double)n;
        for (int i = 0; i < n; ++i) {
          const double d = z[ix[i]] - zb;
          sxx = fma(d, d, sxx); sxy = fma(d, sY[ix[i]] - yb, sxy);
        }
        pi = sxy / sxx;
        const double al = yb - pi * zb;
        for (int i = 0; i < n; ++i) {
          const double zi = z[ix[i]];
          sH[i] = (sY[ix[i]] - al - pi * zi) * (zi - zb) / sxx;
        }
        double V = 0.0;
        for (int i = 0; i < n; ++i) V = fma(sH[i], sH[i], V);
        for (int j = 1; j <= q && j < n; ++j) {
          double c = 0.0;
          for (int i = 0; i + j < n; ++i) c = fma(sH[i], sH[i + j], c);
          V = fma(2.0 * (1.0 - (double)j / (double)(q + 1)), c, V);
        }
        Fs = pi * pi / V;
      }
      double* o = om + bk * (size_t)(n_boot + 1) * r;
      for (int a = 0; a < r; ++a) o[a] = code == 0 ? sG[a] : DFM_NAN;
      nk[bk] = n; ist[bk] = code; red[2] = (double)code;
      if (nobs) nobs[bk] = n;
      if (rel) rel[bk] = rho2;
      if (fpi) fpi[bk] = pi;
      if (fF) fF[bk] = Fs;
    }
    DFM_SYNC();
    const bool ok = (int)red[2] == 0;
    if (eps)
      for (int t = DFM_TID; t < Tp; t += DFM_NT) {
        double e = 0.0;
        for (int a = 0; a < r; ++a) e = fma(sG[a], Ub[t + (size_t)Tp * a], e);
        eps[bk * Tp + t] = ok && !sBad[t] ? e : DFM_NAN;
      }
    DFM_SYNC();                                        // (sG and red are rewritten by the next instrument)
  }
}

// Shared memory of k_iv_boot: the compacted u (r x Tp at most) and z (Tp), the replicates' sums (r IV_BT).
__host__ __device__ inline size_t iv_boot_smem_bytes(int r, int Tp) {
  return ((size_t)Tp * (r + 1) + (size_t)r * IV_BT) * 8;
}

// grid (ceil(n_boot / IV_BT), B ni), IV_BT threads.  Replicate rho = 1 + x IV_BT + t of (model, instrument) bk = y: the n = nk[bk]
// periods of T_k indexed 0 .. n-1, block length l = min(block, n), nbl = ceil(n / l) block starts s_j = floor(u_j (n - l + 1)),
// u_j the uniform number (rho ni + k) Tp + j of the Philox stream of ids[b], tag 20; the blocks concatenated and cut at n;
// zbar*, g* = (1/n) sum u*_i (z*_i - zbar*), om[(bk (1 + n_boot) + rho) r ..] = g* / |g*| (NaN when g* = 0 or ist[bk] != 0).
__global__ void k_iv_boot(const double* __restrict__ U, const double* __restrict__ Z, const int* __restrict__ idx,
                          const int* __restrict__ nk, const int* __restrict__ ist, int r, int Tp, int ni, int block, int n_boot,
                          unsigned long long seed, const unsigned long long* __restrict__ ids, double* __restrict__ om) {
  DFM_SMEM(sm);
  const int bk = DFM_BY, b = bk / ni, kk = bk % ni;
  const int n = nk[bk];
  const bool bad = ist[bk] != 0;
  double* sU = sm;                                     // [a][i]  u of period i of T_k
  double* sZ = sU + (size_t)r * n;                     // [i]
  double* acc = sZ + n;                                // [a][IV_BT]
  if (!bad) {
    const int* ix = idx + (size_t)bk * Tp;
    const double* Ub = U + (size_t)b * Tp * r;
    for (int e = DFM_TID; e < r * n; e += DFM_NT) { const int a = e / n, i = e % n; sU[e] = Ub[ix[i] + (size_t)Tp * a]; }
    for (int i = DFM_TID; i < n; i += DFM_NT) sZ[i] = Z[(size_t)Tp * kk + ix[i]];
  }
  DFM_SYNC();
  const int l = block < n ? block : n, nbl = bad ? 0 : (n + l - 1) / l, span = n - l + 1;
  const unsigned long long id = ids[b];
  for (int tl = DFM_TID; tl < IV_BT; tl += DFM_NT) {
    const long long rho = 1 + (long long)DFM_BX * IV_BT + tl;
    if (rho > n_boot) continue;
    double* o = om + ((size_t)bk * (n_boot + 1) + (size_t)rho) * r;
    if (bad) { for (int a = 0; a < r; ++a) o[a] = DFM_NAN; continue; }
    const unsigned long long e0 = ((unsigned long long)rho * ni + kk) * (unsigned long long)Tp;
    double zs = 0.0;
    for (int j = 0, c = 0; j < nbl; ++j) {
      const int s = (int)(rng_uniform(seed, id, RNG_PROXY, e0 + j) * span);
      for (int i = 0; i < l && c < n; ++i, ++c) zs += sZ[s + i];
    }
    const double zb = zs / (double)n;
    double* ac = acc + tl;
    for (int a = 0; a < r; ++a) ac[(size_t)a * IV_BT] = 0.0;
    for (int j = 0, c = 0; j < nbl; ++j) {
      const int s = (int)(rng_uniform(seed, id, RNG_PROXY, e0 + j) * span);
      for (int i = 0; i < l && c < n; ++i, ++c) {
        const double d = sZ[s + i] - zb;
        for (int a = 0; a < r; ++a) ac[(size_t)a * IV_BT] = fma(sU[(size_t)a * n + s + i], d, ac[(size_t)a * IV_BT]);
      }
    }
    double nrm2 = 0.0;
    for (int a = 0; a < r; ++a) { const double g = ac[(size_t)a * IV_BT] / (double)n; ac[(size_t)a * IV_BT] = g; nrm2 = fma(g, g, nrm2); }
    const bool ok = nrm2 > 0.0 && nrm2 < INFINITY;
    const double inv = 1.0 / sqrt(nrm2);
    for (int a = 0; a < r; ++a) o[a] = ok ? ac[(size_t)a * IV_BT] * inv : DFM_NAN;
  }
}

// Shared memory of k_iv_rot: Omega (r r), v (r), and the three scalars sc[0 .. 2].
__host__ __device__ inline size_t iv_rot_smem_bytes(int r) { return ((size_t)r * r + r + 3) * 8; }

// grid (nrec), 64 threads, shared iv_rot_smem_bytes(r).  Record s is (model, instrument, replicate) g = g0 + s of the chunk's
// record order (bk = g / (1 + n_boot)); omega = om[g r ..].  Omega = -sigma (I - 2 v v' / v'v), v = omega + sigma e_1,
// sigma = +1 when omega_0 >= 0 and -1 otherwise: orthogonal, first column omega.  rec[s][j][h][a] = (Psi_h Omega)_{a j} (k_irf's
// layout, for k_series_resp; Psi of model bk / ni), sst[s] = 0, or 3 (NaN record) when omega is NaN.
__global__ void k_iv_rot(const double* __restrict__ irf, const double* __restrict__ om, long long g0, int r, int H, int ni, int n_boot,
                         double* __restrict__ rec, int* __restrict__ sst) {
  DFM_SMEM(sm);
  const int s = DFM_BX;
  const long long g = g0 + s;
  const long long bk = g / (n_boot + 1);
  const double* w = om + (size_t)g * r;
  double* sQ = sm;                                     // [j][a] Omega
  double* v = sQ + (size_t)r * r;
  double* sc = v + r;                                  // [0] 2 / v'v  [1] -sigma  [2] bad
  if (DFM_TID == 0) {
    bool bad = false;
    for (int a = 0; a < r; ++a) bad = bad || is_nan(w[a]);
    const double sg = w[0] >= 0.0 ? 1.0 : -1.0;
    double vv = 0.0;
    for (int a = 0; a < r; ++a) { v[a] = w[a] + (a == 0 ? sg : 0.0); vv = fma(v[a], v[a], vv); }
    sc[0] = 2.0 / vv; sc[1] = -sg; sc[2] = bad ? 1.0 : 0.0;
  }
  DFM_SYNC();
  const bool bad = sc[2] != 0.0;
  for (int e = DFM_TID; e < r * r; e += DFM_NT) {
    const int a = e % r, j = e / r;
    sQ[e] = sc[1] * ((a == j ? 1.0 : 0.0) - sc[0] * v[a] * v[j]);
  }
  DFM_SYNC();
  if (DFM_TID == 0 && !bad) for (int a = 0; a < r; ++a) sQ[a] = w[a];    // column 0 exactly omega
  DFM_SYNC();
  const double* P = irf + (size_t)(bk / ni) * r * r * H;
  double* Ro = rec + (size_t)s * r * r * H;
  for (int e = DFM_TID; e < r * r * H; e += DFM_NT) {
    const int a = e % r, h = (e / r) % H, j = e / (r * H);
    double x = 0.0;
    for (int l = 0; l < r; ++l) x = fma(P[((size_t)l * H + h) * r + a], sQ[(size_t)j * r + l], x);
    Ro[e] = bad ? DFM_NAN : x;
  }
  if (DFM_TID == 0) sst[s] = bad ? 3 : 0;
}

}  // namespace dfm
