// dfm_kernels_resp.cuh -- series responses and forecast-error variance decompositions of many state-space models at once
// (dfm_series_responses).  Per model (Lam, R, A, Q), L = chol(Q), Psi_h = [M^h]_{1:r,1:r} L (h = 0 .. H-1) and
// c_{i,h} = lam_i' Psi_h:
//   k_sr_prep       one CTA per model: M (companion of A), Qsel = [I 0], G = [L; 0] for k_irf, and the model's status
//   k_irf           (dfm_kernels_np.cuh) Psi_h e_j for every shock j < r
//   k_series_resp   one thread per (series, model): resp[i,h,j] = scale_i c_{i,h,j} and
//                   fevd[i,h,j] = sum_{l<=h} c_{i,l,j}^2 / (sum_{l<=h} |c_{i,l}|^2 + R_i) for the leading n_shock shocks
// The spec is tests/identified_oracle.py.  k_series_resp is plain FMA code with coalesced stores (consecutive threads write
// consecutive series), so the host-emulation build runs the same source.
#pragma once
#include "dfm_common.cuh"

namespace dfm {

#define SR_NS 128              // series (threads) per CTA of k_series_resp

// M, Qsel, G of each model for k_irf; status[b] = 3 when A or Q holds a NaN (a failed chain) or Q is not positive definite.
// grid (B), 64 threads, shared r r + 8 doubles.
__global__ void k_sr_prep(const double* __restrict__ Aall, const double* __restrict__ Qall, int r, int p, double* __restrict__ Mall,
                          double* __restrict__ Qsel, double* __restrict__ Gall, int* __restrict__ status) {
  DFM_SMEM(sm);
  const int b = DFM_BX, k = r * p;
  const double* A = Aall + (size_t)b * r * k;
  const double* Q = Qall + (size_t)b * r * r;
  double* S = sm;
  int* info = (int*)(S + r * r);
  if (DFM_TID == 0) { info[0] = 0; info[1] = 0; }
  DFM_SYNC();
  for (int e = DFM_TID; e < r * r; e += DFM_NT) { S[e] = Q[e]; if (is_nan(Q[e])) info[1] = 1; }
  for (int e = DFM_TID; e < r * k; e += DFM_NT) if (is_nan(A[e])) info[1] = 1;
  DFM_SYNC();
  if (!info[1]) bm_chol(S, r, r, info);
  DFM_SYNC();
  const bool bad = info[0] || info[1];
  double* M = Mall + (size_t)b * k * k;
  for (int e = DFM_TID; e < k * k; e += DFM_NT) {
    const int i = e % k, j = e / k;
    M[e] = i < r ? A[i + (size_t)r * j] : (j == i - r ? 1.0 : 0.0);
  }
  double* Qs = Qsel + (size_t)b * r * k;
  for (int e = DFM_TID; e < r * k; e += DFM_NT) { const int i = e % r, j = e / r; Qs[e] = i == j ? 1.0 : 0.0; }
  double* G = Gall + (size_t)b * k * r;
  for (int e = DFM_TID; e < k * r; e += DFM_NT) {
    const int i = e % k, j = e / k;
    G[e] = bad ? DFM_NAN : (i < r && i >= j ? S[i + r * j] : 0.0);
  }
  if (DFM_TID == 0) status[b] = bad ? 3 : 0;
}

// Horizons of Psi staged per pass of k_series_resp: (r + n_shock + 1) SR_NS + hc r r doubles of shared memory.
__host__ __device__ inline size_t series_resp_smem_doubles(int r, int ns, int hc) {
  return (size_t)(r + ns + 1) * SR_NS + (size_t)hc * r * r;
}

// grid (ceil(N / SR_NS), B), SR_NS threads.  Lam N x r, R N per model, record b reading model b / ldiv (ldiv = 1: one record per
// model; dfm_sign_restrictions: n_keep rotated records per model); scale N (NULL: 1); irf: k_irf's records of all r shocks,
// [b][j][h][a] = (Psi_h)_{a j}; st: the records' status.  resp / fevd (may be NULL): N x H x ns per model, column-major.  The
// CTA stages its series' loadings, then Psi in passes of hc horizons; per series the running FEV sums of its ns leading shocks
// sit in shared memory, the running total in sD.
__global__ void k_series_resp(const double* __restrict__ Lam, const double* __restrict__ R, const double* __restrict__ scale,
                              const double* __restrict__ irf, const int* __restrict__ st, int N, int r, int H, int ns, int hc,
                              int ldiv, double* __restrict__ resp, double* __restrict__ fevd) {
  DFM_SMEM(sm);
  const int b = DFM_BY, i0 = DFM_BX * SR_NS;
  double* sL = sm;                                     // [r][SR_NS]  loadings, NaN: series out of the model or past N
  double* cum = sL + (size_t)r * SR_NS;                // [ns][SR_NS] sum_{l<=h} c_{i,l,j}^2
  double* sD = cum + (size_t)ns * SR_NS;               // [SR_NS]     sum_{l<=h} |c_{i,l}|^2
  double* sP = sD + SR_NS;                             // [r][hc][r]  Psi of the pass
  const bool bad = st[b] != 0;
  const size_t bm = (size_t)(b / ldiv);
  const double* Lb = Lam + bm * N * r;
  const double* P = irf + (size_t)b * r * r * H;
  const size_t o0 = (size_t)b * N * H * ns;
  for (int e = DFM_TID; e < r * SR_NS; e += DFM_NT) {
    const int a = e / SR_NS, i = i0 + e % SR_NS;
    sL[e] = i < N ? Lb[i + (size_t)N * a] : DFM_NAN;
  }
  for (int e = DFM_TID; e < (ns + 1) * SR_NS; e += DFM_NT) cum[e] = 0.0;
  for (int h0 = 0; h0 < H; h0 += hc) {
    const int nh = H - h0 < hc ? H - h0 : hc;
    DFM_SYNC();
    for (int e = DFM_TID; e < r * nh * r; e += DFM_NT) {
      const int a = e % r, hl = (e / r) % nh, j = e / (r * nh);
      sP[e] = P[((size_t)j * H + h0 + hl) * r + a];
    }
    DFM_SYNC();
    for (int il = DFM_TID; il < SR_NS; il += DFM_NT) {
      const int i = i0 + il;
      if (i >= N) continue;
      const double Ri = R[bm * N + i], sc = scale ? scale[i] : 1.0;
      bool in = !bad && !is_nan(Ri);
      for (int a = 0; a < r; ++a) if (is_nan(sL[(size_t)a * SR_NS + il])) in = false;
      double den = sD[il];
      for (int hl = 0; hl < nh; ++hl) {
        const size_t oh = o0 + i + (size_t)N * (h0 + hl);
        for (int j = 0; j < r; ++j) {
          const double* pj = sP + ((size_t)j * nh + hl) * r;
          double c = 0.0;
          for (int a = 0; a < r; ++a) c += sL[(size_t)a * SR_NS + il] * pj[a];
          den += c * c;
          if (j < ns) {
            cum[(size_t)j * SR_NS + il] += c * c;
            if (resp) resp[oh + (size_t)N * H * j] = in ? sc * c : DFM_NAN;
          }
        }
        if (fevd)
          for (int j = 0; j < ns; ++j) fevd[oh + (size_t)N * H * j] = in ? cum[(size_t)j * SR_NS + il] / (den + Ri) : DFM_NAN;
      }
      sD[il] = den;
    }
  }
}

}  // namespace dfm
