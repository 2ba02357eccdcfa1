// dfm_kernels_hd.cuh -- historical decompositions of many state-space models at once (dfm_historical_decomposition).  Per
// model (Lam, R, A, Q) and factor path f_0 .. f_{Tp-1}, L = chol(Q): the structural shocks eps_t = L^-1 (f_t - sum_l A_l f_{t-l})
// and the split of lam_i' f_t into the part carried over from the base row t0 and the parts due to each leading shock and
// to the remaining shocks (include/dfm_b200.h has the definitions):
//   k_sr_prep     (dfm_kernels_resp.cuh) one CTA per model: M (companion of A), G = [L; 0] and the model's status
//   k_hd_paths    one CTA per model: eps (parallel over t), then nc = n_shock + 2 factor-level recursions (base, each leading
//                 shock, the rest) y_t = sum_l A_l y_{t-l} + L[:, J] eps_{J,t}, parallel over (recursion, component)
//   k_hd_series   one thread per (series, model): scale_i lam_i' y_{c,t} for every recursion c and row t, consecutive threads
//                 on consecutive series
// Because M is a companion matrix, [M^h z]_{1:r} obeys the r-dimensional recursion above: O(r k) per step, not O(k^2).  The
// spec is tests/history_oracle.py, which takes the other road (the Psi convolution written out).  Plain FMA code, so the
// host-emulation build runs the same source.
#pragma once
#include "dfm_common.cuh"

namespace dfm {

#define HD_NS 64               // series (threads) per CTA of k_hd_series
#define HD_PT 128              // threads per CTA of k_hd_paths

// Shared memory of k_hd_paths: A (r k), L (r r), the ring of the last p + 1 rows of every recursion (nc (p + 1) r), a flag.
__host__ __device__ inline size_t hd_paths_smem_doubles(int r, int p, int nc) {
  return (size_t)r * r * p + (size_t)r * r + (size_t)nc * (p + 1) * r + 1;
}

// grid (B), HD_PT threads.  M, G, st: k_sr_prep's records (G = [L; 0], k x r); F: Tp x r per model.  eps (Tp x r per model,
// NaN for t < p) and Y (the recursions, [t][c][a] per model: c = 0 base, 1 .. ns the leading shocks, ns + 1 the rest) are
// written; st[b] becomes 3 when the path holds a NaN.  A bad model gets NaN eps and leaves Y unwritten (k_hd_series does not
// read it).
__global__ void k_hd_paths(const double* __restrict__ Mall, const double* __restrict__ Gall, const double* __restrict__ Fall,
                           int r, int p, int Tp, int t0, int ns, int* __restrict__ st, double* eps, double* __restrict__ Yall) {
  DFM_SMEM(sm);
  const int b = DFM_BX, k = r * p, nc = ns + 2;
  const double* M = Mall + (size_t)b * k * k;
  const double* G = Gall + (size_t)b * k * r;
  const double* F = Fall + (size_t)b * Tp * r;
  double* E = eps + (size_t)b * Tp * r;
  double* Y = Yall + (size_t)b * nc * Tp * r;
  double* sA = sm;                                     // [r][k]  A (column-major, ld r)
  double* sL = sA + (size_t)r * k;                     // [r][r]  L
  double* ring = sL + (size_t)r * r;                   // [nc][p + 1][r]  y_s at slot s mod (p + 1)
  int* flag = (int*)(ring + (size_t)nc * (p + 1) * r);
  if (DFM_TID == 0) *flag = st[b] != 0;
  DFM_SYNC();
  for (int e = DFM_TID; e < Tp * r; e += DFM_NT) if (is_nan(F[e])) *flag = 1;
  for (int e = DFM_TID; e < r * k; e += DFM_NT) sA[e] = M[e % r + (size_t)k * (e / r)];
  for (int e = DFM_TID; e < r * r; e += DFM_NT) sL[e] = G[e % r + (size_t)k * (e / r)];
  DFM_SYNC();
  if (*flag) {
    for (int e = DFM_TID; e < Tp * r; e += DFM_NT) E[e] = DFM_NAN;
    if (DFM_TID == 0) st[b] = 3;
    return;
  }
  // eps_t = L^-1 u_t, u_t = f_t - sum_l A_l f_{t-l}: one thread per period, u and the forward substitution in place in E
  for (int t = DFM_TID; t < Tp; t += DFM_NT) {
    if (t < p) { for (int a = 0; a < r; ++a) E[t + (size_t)Tp * a] = DFM_NAN; continue; }
    for (int a = 0; a < r; ++a) {
      double u = F[t + (size_t)Tp * a];
      for (int l = 1; l <= p; ++l)
        for (int c = 0; c < r; ++c) u -= sA[a + (size_t)r * ((l - 1) * r + c)] * F[t - l + (size_t)Tp * c];
      for (int c = 0; c < a; ++c) u -= sL[a + (size_t)r * c] * E[t + (size_t)Tp * c];
      E[t + (size_t)Tp * a] = u / sL[a + (size_t)r * a];
    }
  }
  // rows t <= t0: base = f_t, the shock parts 0; the ring holds y_{t0-p+1} .. y_t0
  for (int e = DFM_TID; e < nc * (t0 + 1) * r; e += DFM_NT) {
    const int a = e % r, t = (e / r) % (t0 + 1), c = e / (r * (t0 + 1));
    const double v = c == 0 ? F[t + (size_t)Tp * a] : 0.0;
    Y[((size_t)t * nc + c) * r + a] = v;
    if (t > t0 - p) ring[((size_t)c * (p + 1) + t % (p + 1)) * r + a] = v;
  }
  DFM_SYNC();                                          // (E and the ring complete)
  for (int t = t0 + 1; t < Tp; ++t) {
    const int w = t % (p + 1);
    for (int e = DFM_TID; e < nc * r; e += DFM_NT) {
      const int a = e % r, c = e / r;
      const double* yc = ring + (size_t)c * (p + 1) * r;
      double v = 0.0;
      for (int l = 1; l <= p; ++l) {
        const double* yl = yc + (size_t)((t - l) % (p + 1)) * r;
        const double* Al = sA + (size_t)r * (l - 1) * r + a;
        for (int j = 0; j < r; ++j) v += Al[(size_t)r * j] * yl[j];
      }
      if (c >= 1 && c <= ns) v += sL[a + (size_t)r * (c - 1)] * E[t + (size_t)Tp * (c - 1)];
      else if (c == ns + 1) for (int j = ns; j <= a; ++j) v += sL[a + (size_t)r * j] * E[t + (size_t)Tp * j];
      ring[((size_t)c * (p + 1) + w) * r + a] = v;     // (slot w holds y_{t-p-1}, which no thread reads at step t)
      Y[((size_t)t * nc + c) * r + a] = v;
    }
    DFM_SYNC();
  }
}

// Shared memory of k_hd_series: the loadings (r HD_NS; registers hold them during the products) and tc rows of the recursions.
__host__ __device__ inline size_t hd_series_smem_doubles(int r, int nc, int tc) {
  return (size_t)r * HD_NS + (size_t)tc * nc * r;
}

// grid (ceil(N / HD_NS), B), HD_NS threads, RM >= r.  Lam N x r, R N per model; scale N (NULL: 1); Y, st: k_hd_paths' records.
// contrib (N x Tp x ns), rest, base (N x Tp) per model, column-major, any may be NULL.  The CTA stages its series' loadings,
// then the recursions in passes of tc rows; each thread keeps its loadings in registers and writes scale_i lam_i' y_{c,t}.
template <int RM>
__global__ void k_hd_series(const double* __restrict__ Lam, const double* __restrict__ R, const double* __restrict__ scale,
                            const double* __restrict__ Yall, const int* __restrict__ st, int N, int r, int Tp, int ns, int tc,
                            double* __restrict__ contrib, double* __restrict__ rest, double* __restrict__ base) {
  DFM_SMEM(sm);
  const int b = DFM_BY, i0 = DFM_BX * HD_NS, nc = ns + 2;
  double* sLm = sm;                                    // [r][HD_NS]   loadings, NaN past N
  double* sY = sLm + (size_t)r * HD_NS;                // [tl][c][a]   rows tp .. tp + tc - 1 of the recursions
  const bool bad = st[b] != 0;
  const double* Lb = Lam + (size_t)b * N * r;
  const double* Y = Yall + (size_t)b * nc * Tp * r;
  const size_t o0 = (size_t)b * N * Tp, oc = o0 * ns;
  for (int e = DFM_TID; e < r * HD_NS; e += DFM_NT) {
    const int a = e / HD_NS, i = i0 + e % HD_NS;
    sLm[e] = i < N ? Lb[i + (size_t)N * a] : DFM_NAN;
  }
  DFM_SYNC();
  for (int il = DFM_TID; il < HD_NS; il += DFM_NT) {
    const int i = i0 + il;
    if (i >= N) continue;
    bool in = !bad && !is_nan(R[(size_t)b * N + i]);
    for (int a = 0; a < r; ++a) if (is_nan(sLm[(size_t)a * HD_NS + il])) in = false;
    if (in) continue;
    for (int t = 0; t < Tp; ++t) {                     // out of the model, or a failed model: NaN columns
      if (base) base[o0 + i + (size_t)N * t] = DFM_NAN;
      if (rest) rest[o0 + i + (size_t)N * t] = DFM_NAN;
      if (contrib) for (int j = 0; j < ns; ++j) contrib[oc + i + (size_t)N * t + (size_t)N * Tp * j] = DFM_NAN;
    }
  }
  if (bad) return;
  for (int tp = 0; tp < Tp; tp += tc) {
    const int nt = Tp - tp < tc ? Tp - tp : tc;
    DFM_SYNC();
    const double* Yp = Y + (size_t)tp * nc * r;         // (rows tp .. tp + nt - 1 are contiguous)
    for (int e = DFM_TID; e < nt * nc * r; e += DFM_NT) sY[e] = Yp[e];
    DFM_SYNC();
    for (int il = DFM_TID; il < HD_NS; il += DFM_NT) {
      const int i = i0 + il;
      if (i >= N) continue;
      double lam[RM];
      bool in = !is_nan(R[(size_t)b * N + i]);
#pragma unroll
      for (int a = 0; a < RM; ++a) {
        lam[a] = a < r ? sLm[(size_t)a * HD_NS + il] : 0.0;
        if (is_nan(lam[a])) in = false;
      }
      if (!in) continue;
      const double sc = scale ? scale[i] : 1.0;
      for (int tl = 0; tl < nt; ++tl) {
        const size_t ot = i + (size_t)N * (tp + tl);
        const double* yt = sY + (size_t)tl * nc * r;
        for (int c = 0; c < nc; ++c) {
          const double* y = yt + (size_t)c * r;
          double v = 0.0;
#pragma unroll
          for (int a = 0; a < RM; ++a) if (a < r) v += lam[a] * y[a];
          v *= sc;
          if (c == 0) { if (base) base[o0 + ot] = v; }
          else if (c <= ns) { if (contrib) contrib[oc + ot + (size_t)N * Tp * (c - 1)] = v; }
          else if (rest) rest[o0 + ot] = v;
        }
      }
    }
  }
}

}  // namespace dfm
