// dfm_kernels_narr.cuh -- narrative sign restrictions (dfm_narrative_sign_restrictions): the sign-restriction search of
// dfm_kernels_sign.cuh with statements about dated episodes added, and the importance weight of every kept draw.  Per model,
// on top of 4.14's L, Psi_h and c_{i,h}: the orthonormalised reduced-form shocks u_t = L^-1 (f_t - sum_l A_l f_{t-l}) of a
// factor path, the structural shocks eps~_t = Omega' u_t, and the contribution of shock k to series i over t .. t+h,
// H_{i,k}(t, h) = omega_k' G omega_k with G = sum_{l<=h} c_{i,l}' u_{t+h-l}' (include/dfm_b200.h has the definition):
//   k_sr_prep, k_irf, k_sign_prep  (reused) Psi_h, the sign rows' s c_{i,h}, the pick state
//   k_narr_prep    one CTA per model: u_t, and per narrative row s u_t (kind 0) or the r x r matrix (s) G (kinds 1-3)
//   k_narr_cand    one thread per candidate: k_sign_cand's column routine, each shock's sign rows and narrative rows tested by
//                  nr_orient, then (kinds 1 and 2 only) the remaining columns and the share rows; one accept bit per candidate
//   k_sign_pick    (reused) the accept count and the first n_keep ids
//   k_narr_rot     one CTA per kept slot: Omega rebuilt with the same routines (the same bits and flips), the records Psi_h Omega
//                  for k_series_resp, and the kept draw's structural shock path
//   k_narr_omega   one thread per simulation: the narrative rows evaluated on N(0, I) shocks -> n_ok per kept slot
//   k_narr_weight  weight = n_sim / n_ok
//   k_wpercentiles weighted percentiles (the first record whose exact cumulative weight reaches q / 100 of the total)
// H is quadratic in omega_k, so the kinds 1-3 do not depend on a column's orientation; only kind 0 joins the flip rule.
// Explicit fma in every decision, so k_narr_cand and k_narr_rot take the same decisions.  The spec is tests/narrative_oracle.py.
#pragma once
#include "dfm_common.cuh"
#include "dfm_kernels_sign.cuh"

#ifdef DFM_EMU
static inline unsigned long long atomicAdd(unsigned long long* p, unsigned long long v) { unsigned long long o = *p; *p += v; return o; }
#endif

namespace dfm {

enum { RNG_NARR = 19 };        // e_{k,tau} of simulation s of model id: element (s nP + p) r + k, p the position of tau

#define NR_NMAX 64             // narrative rows bound
#define NR_SIMT 128            // simulations (threads) per CTA of k_narr_omega
#define NR_PT 128              // threads per CTA of k_narr_prep

// One narrative row as the kernels see it: kind (0 shock sign, 1 most important, 2 overwhelming, 3 contribution sign), shock
// j (0-based), series i, row t, window h, sign s, the offset of its data in the model's block D (r doubles for kind 0, r^2
// otherwise), the position of t in the sorted union of the rows' periods, and the offset of its c omega block in
// k_narr_omega's shared memory ((h + 1) r doubles, kinds 1-3).
struct nr_row { int kind, shock, series, t, h, sign, doff, pos, coff; };

// v = w' G w (G r x r row-major [a][b], w at stride s)
__device__ __forceinline__ double nr_quad(const double* G, const double* w, int s, int r) {
  double v = 0.0;
  for (int a = 0; a < r; ++a) {
    double g = 0.0;
    for (int b = 0; b < r; ++b) g = fma(G[(size_t)a * r + b], w[(size_t)b * s], g);
    v = fma(w[(size_t)a * s], g, v);
  }
  return v;
}

// Test and orient column omega_j (w, stride s): Cr / nsg its sign rows (s c, as sg_test), rows[0 .. nn) its narrative rows of
// kinds 0 and 3, D the model's narrative block.  The sign rows fix the orientation when there are any (4.14's rule) and the
// kind-0 rows are tested at it; otherwise the kind-0 rows are the flip group (all > 0 keep, all < 0 flip).  Kind-3 rows are
// tested as they are (H does not depend on the orientation).  +1 keep, -1 flip, 0 rejected.
__device__ __forceinline__ int nr_orient(const double* Cr, int nsg, const nr_row* rows, int nn, const double* D, const double* w,
                                         int s, int r) {
  int f = 1;
  if (nsg > 0) { f = sg_test(Cr, nsg, w, s, r); if (f == 0) return 0; }
  bool pos = true, neg = true;
  for (int q = 0; q < nn; ++q) {
    if (rows[q].kind != 0) continue;
    const double* u = D + rows[q].doff;
    double v = 0.0;
    for (int a = 0; a < r; ++a) v = fma(u[a], w[(size_t)a * s], v);
    pos = pos && v > 0.0;
    neg = neg && v < 0.0;
  }
  if (nsg == 0) f = pos ? 1 : (neg ? -1 : 0);
  else if (!(f > 0 ? pos : neg)) f = 0;
  if (f == 0) return 0;
  for (int q = 0; q < nn; ++q)
    if (rows[q].kind == 3 && !(nr_quad(D + rows[q].doff, w, s, r) > 0.0)) return 0;
  return f;
}

// Kinds 1 and 2: |H_j| > max_{k != j} |H_k| (most important) or > sum_{k != j} |H_k| (overwhelming), over all r columns of Q
// (column k, element a at Q[(k r + a) s]).
__device__ __forceinline__ bool nr_share(const nr_row& row, const double* D, const double* Q, int s, int r) {
  double hj = 0.0, mx = 0.0, sum = 0.0;
  for (int k = 0; k < r; ++k) {
    const double v = fabs(nr_quad(D + row.doff, Q + (size_t)k * r * s, s, r));
    if (k == row.shock) hj = v;
    else { mx = v > mx ? v : mx; sum += v; }
  }
  return row.kind == 1 ? hj > mx : hj > sum;
}

// grid (B), NR_PT threads, shared (r k + r r + 1) doubles.  M, G, st: k_sr_prep's records; irf: k_irf's; F: Tp x r per model
// (column-major).  U[b] = u_t ([t][a], NaN for t < p); D[b] (nD doubles): each row's s u_t or (s) G ([a][b]).  st[b] becomes
// 3 when the path holds a NaN, otherwise DFM_ERR_ARG when a narrative series is out of the model (NaN loading row or R_i); a
// model that k_sr_prep or k_sign_prep already failed keeps its status; a bad model leaves U and D unwritten.
__global__ void k_narr_prep(const double* __restrict__ Lam, const double* __restrict__ R, const double* __restrict__ irf,
                            const double* __restrict__ Mall, const double* __restrict__ Gall, const double* __restrict__ Fall, int N,
                            int r, int p, int H, int Tp, int nN, const nr_row* __restrict__ rows, int nD, int* __restrict__ st,
                            double* __restrict__ Uall, double* __restrict__ Dall) {
  DFM_SMEM(sm);
  const int b = DFM_BX, k = r * p;
  const double* M = Mall + (size_t)b * k * k;
  const double* G = Gall + (size_t)b * k * r;
  const double* F = Fall + (size_t)b * Tp * r;
  const double* Lb = Lam + (size_t)b * N * r;
  const double* P = irf + (size_t)b * r * r * H;
  double* U = Uall + (size_t)b * Tp * r;
  double* D = Dall + (size_t)b * nD;
  double* sA = sm;                                     // [r][k]  A (column-major, ld r)
  double* sL = sA + (size_t)r * k;                     // [r][r]  L
  int* flag = (int*)(sL + (size_t)r * r);              // [0] a narrative series out of the model, [1] a NaN path row
  if (DFM_TID == 0) {
    int fl = 0;
    for (int q = 0; q < nN; ++q) {
      if (rows[q].kind == 0) continue;
      const int i = rows[q].series;
      bool bad = is_nan(R[(size_t)b * N + i]);
      for (int a = 0; a < r; ++a) bad = bad || is_nan(Lb[i + (size_t)N * a]);
      if (bad) fl = 1;
    }
    flag[0] = fl;
    flag[1] = 0;
  }
  DFM_SYNC();
  if (st[b] != 0) return;
  for (int e = DFM_TID; e < Tp * r; e += DFM_NT) if (is_nan(F[e])) flag[1] = 1;
  for (int e = DFM_TID; e < r * k; e += DFM_NT) sA[e] = M[e % r + (size_t)k * (e / r)];
  for (int e = DFM_TID; e < r * r; e += DFM_NT) sL[e] = G[e % r + (size_t)k * (e / r)];
  DFM_SYNC();
  const int fl = flag[1] ? 3 : (flag[0] ? DFM_ERR_ARG : 0);     // (a NaN path row ranks first, as the sign rows' checks)
  DFM_SYNC();
  if (fl) {
    if (DFM_TID == 0) st[b] = fl;
    return;
  }
  // u_t = L^-1 (f_t - sum_l A_l f_{t-l}): one thread per period, forward substitution in place
  for (int t = DFM_TID; t < Tp; t += DFM_NT) {
    double* ut = U + (size_t)t * r;
    if (t < p) { for (int a = 0; a < r; ++a) ut[a] = DFM_NAN; continue; }
    for (int a = 0; a < r; ++a) {
      double v = F[t + (size_t)Tp * a];
      for (int l = 1; l <= p; ++l)
        for (int c = 0; c < r; ++c) v -= sA[a + (size_t)r * ((l - 1) * r + c)] * F[t - l + (size_t)Tp * c];
      for (int c = 0; c < a; ++c) v -= sL[a + (size_t)r * c] * ut[c];
      ut[a] = v / sL[a + (size_t)r * a];
    }
  }
  DFM_SYNC();
  for (int q = 0; q < nN; ++q) {
    const nr_row w = rows[q];
    double* Dq = D + w.doff;
    if (w.kind == 0) {
      for (int a = DFM_TID; a < r; a += DFM_NT) Dq[a] = w.sign * U[(size_t)w.t * r + a];
      continue;
    }
    // G[a][c] = sum_l c_{i,l,a} u_{t+h-l,c},  c_{i,l,a} = lam_i' (Psi_l)_{:,a}
    const double sg = w.kind == 3 ? (double)w.sign : 1.0;
    for (int e = DFM_TID; e < r * r; e += DFM_NT) {
      const int a = e / r, c = e % r;
      double v = 0.0;
      for (int l = 0; l <= w.h; ++l) {
        const double* pa = P + ((size_t)a * H + l) * r;
        double cl = 0.0;
        for (int m = 0; m < r; ++m) cl += Lb[w.series + (size_t)N * m] * pa[m];
        v += cl * U[(size_t)(w.t + w.h - l) * r + c];
      }
      Dq[e] = sg * v;
    }
  }
}

// Shared memory of k_narr_cand: the candidates' columns 0 .. ncol-1 and a scratch column (ncol + 1) r SG_NT as k_sign_cand,
// the sign rows nR r, the narrative block nD, the rows, the sign and narrative offsets.
__host__ __device__ inline size_t narr_cand_smem_bytes(int ncol, int r, int nT, int nR, int nD, int nN) {
  return ((size_t)(ncol + 1) * r * SG_NT + (size_t)nR * r + (size_t)nD) * 8 + (size_t)nN * sizeof(nr_row) + (size_t)2 * (nT + 1) * 4;
}

// grid (ntile / 2, B), SG_NT threads.  As k_sign_cand, with nT the shocks tested column by column (the last shock with sign
// rows or narrative rows of kinds 0 / 3, + 1) and ncol the columns drawn (r when rows of kinds 1 / 2 exist, else nT).  off:
// nT + 1 sign-row offsets into C; noff: nT + 1 offsets into rows (shock j's rows of kinds 0 / 3), rows[noff[nT] .. nN) of
// kinds 1 / 2.
__global__ void k_narr_cand(const double* __restrict__ C, const int* __restrict__ off, const double* __restrict__ Dall,
                            const nr_row* __restrict__ rows, const int* __restrict__ noff, const int* __restrict__ st, int r, int nR,
                            int nD, int nN, int nT, int ncol, long long c0, long long n_rot, int ntile, unsigned long long seed,
                            const unsigned long long* __restrict__ ids, unsigned* __restrict__ mask) {
  DFM_SMEM(sm);
  const int b = DFM_BY;
  double* sQ = sm;                                     // [(l r + a)][SG_NT]  columns, then the scratch column
  double* sC = sQ + (size_t)(ncol + 1) * r * SG_NT;    // [rho][a]
  double* sD = sC + (size_t)nR * r;                    // the narrative block
  nr_row* sRow = (nr_row*)(sD + nD);
  int* sOff = (int*)(sRow + nN);
  int* sNoff = sOff + nT + 1;
  for (int e = DFM_TID; e < nR * r; e += DFM_NT) sC[e] = C[(size_t)b * nR * r + e];
  for (int e = DFM_TID; e < nD; e += DFM_NT) sD[e] = Dall[(size_t)b * nD + e];
  for (int e = DFM_TID; e < nN; e += DFM_NT) sRow[e] = rows[e];
  for (int e = DFM_TID; e <= nT; e += DFM_NT) { sOff[e] = off[e]; sNoff[e] = noff[e]; }
  DFM_SYNC();
  const bool bad = st[b] != 0;
  const int n12 = nN - sNoff[nT];
  const unsigned long long id = ids[b], rr = (unsigned long long)r * r;
  for (int tl = DFM_TID; tl < SG_NT; tl += DFM_NT) {
    const long long c = c0 + (long long)DFM_BX * SG_NT + tl;
    bool ok = !bad && c < n_rot;
    if (ok) {
      sg_rng g{seed, id, ~0ull, 0.0};
      double* Q = sQ + tl;
      double* W = Q + (size_t)ncol * r * SG_NT;
      for (int j = 0; j < nT && ok; ++j) {
        sg_column(Q, W, SG_NT, r, j, g, (unsigned long long)c * rr + (unsigned long long)r * j);
        ok = nr_orient(sC + (size_t)sOff[j] * r, sOff[j + 1] - sOff[j], sRow + sNoff[j], sNoff[j + 1] - sNoff[j], sD,
                       Q + (size_t)j * r * SG_NT, SG_NT, r) != 0;
      }
      if (ok && n12 > 0) {
        for (int j = nT; j < ncol; ++j) sg_column(Q, W, SG_NT, r, j, g, (unsigned long long)c * rr + (unsigned long long)r * j);
        for (int q = sNoff[nT]; q < nN && ok; ++q) ok = nr_share(sRow[q], sD, Q, SG_NT, r);
      }
    }
    const size_t w = (size_t)b * ntile + (size_t)DFM_BX * (SG_NT / SG_TILE) + tl / SG_TILE;
#ifndef DFM_EMU
    const unsigned m = __ballot_sync(0xffffffffu, ok);
    if (DFM_LANE == 0) mask[w] = m;
#else
    if (tl % SG_TILE == 0) mask[w] = 0u;
    mask[w] |= (unsigned)ok << (tl % SG_TILE);
#endif
  }
}

// Shared memory of k_narr_rot: Omega and a scratch column (r + 1) r, the sign rows nR r, the narrative block nD, the rows,
// the offsets, the flips.
__host__ __device__ inline size_t narr_rot_smem_bytes(int r, int nT, int nR, int nD, int nN) {
  return ((size_t)(r + 1) * r + (size_t)nR * r + (size_t)nD) * 8 + (size_t)nN * sizeof(nr_row) + (size_t)(2 * (nT + 1) + r) * 4;
}

// grid (B n_keep), 64 threads.  As k_sign_rot, with the flips of nr_orient; also eps[s] (Tp x ne, column-major; NULL when ne =
// 0) = the first ne structural shocks Omega' u_t of the kept draw (NaN for t < p), and nok[s] = 0 for k_narr_omega.
__global__ void k_narr_rot(const double* __restrict__ irf, const double* __restrict__ C, const int* __restrict__ off,
                           const double* __restrict__ Dall, const nr_row* __restrict__ rows, const int* __restrict__ noff,
                           const double* __restrict__ Uall, const int* __restrict__ st, const long long* __restrict__ cand, int r, int H,
                           int Tp, int nR, int nD, int nN, int nT, int n_keep, int ne, unsigned long long seed,
                           const unsigned long long* __restrict__ ids, double* __restrict__ rot, double* __restrict__ rec,
                           int* __restrict__ sst, double* __restrict__ eps, unsigned long long* __restrict__ nok) {
  DFM_SMEM(sm);
  const int s = DFM_BX, b = s / n_keep;
  double* sQ = sm;                                     // [j][a] Omega, then the scratch column
  double* sC = sQ + (size_t)(r + 1) * r;
  double* sD = sC + (size_t)nR * r;
  nr_row* sRow = (nr_row*)(sD + nD);
  int* sOff = (int*)(sRow + nN);
  int* sNoff = sOff + nT + 1;
  int* flip = sNoff + nT + 1;
  const long long c = cand[s];
  const bool bad = st[b] != 0 || c < 0;
  if (!bad) {
    for (int e = DFM_TID; e < nR * r; e += DFM_NT) sC[e] = C[(size_t)b * nR * r + e];
    for (int e = DFM_TID; e < nD; e += DFM_NT) sD[e] = Dall[(size_t)b * nD + e];
    for (int e = DFM_TID; e < nN; e += DFM_NT) sRow[e] = rows[e];
    for (int e = DFM_TID; e <= nT; e += DFM_NT) { sOff[e] = off[e]; sNoff[e] = noff[e]; }
    DFM_SYNC();
    if (DFM_TID == 0) {
      sg_rng g{seed, ids[b], ~0ull, 0.0};
      const unsigned long long rr = (unsigned long long)r * r;
      for (int j = 0; j < r; ++j) {
        sg_column(sQ, sQ + (size_t)r * r, 1, r, j, g, (unsigned long long)c * rr + (unsigned long long)r * j);
        flip[j] = j < nT ? nr_orient(sC + (size_t)sOff[j] * r, sOff[j + 1] - sOff[j], sRow + sNoff[j], sNoff[j + 1] - sNoff[j], sD,
                                     sQ + (size_t)j * r, 1, r)
                         : 1;
      }
    }
    DFM_SYNC();
    for (int e = DFM_TID; e < r * r; e += DFM_NT) if (flip[e / r] < 0) sQ[e] = -sQ[e];
    DFM_SYNC();
  }
  if (rot) for (int e = DFM_TID; e < r * r; e += DFM_NT) rot[(size_t)s * r * r + e] = bad ? DFM_NAN : sQ[e];
  const double* P = irf + (size_t)b * r * r * H;
  double* Ro = rec + (size_t)s * r * r * H;
  for (int e = DFM_TID; e < r * r * H; e += DFM_NT) {
    const int a = e % r, h = (e / r) % H, j = e / (r * H);
    double v = 0.0;
    if (!bad) for (int l = 0; l < r; ++l) v += P[((size_t)l * H + h) * r + a] * sQ[(size_t)j * r + l];
    Ro[e] = bad ? DFM_NAN : v;
  }
  if (eps) {
    const double* U = Uall + (size_t)b * Tp * r;
    double* E = eps + (size_t)s * Tp * ne;
    for (int e = DFM_TID; e < Tp * ne; e += DFM_NT) {
      const int t = e % Tp, k = e / Tp;
      double v = 0.0;
      if (!bad) for (int a = 0; a < r; ++a) v = fma(sQ[(size_t)k * r + a], U[(size_t)t * r + a], v);
      E[e] = bad ? DFM_NAN : v;
    }
  }
  if (DFM_TID == 0) { sst[s] = bad ? 3 : 0; nok[s] = 0ull; }
}

// grid (B n_keep, ceil(n_sim / NR_SIMT)), NR_SIMT threads, shared nC doubles + 1 int.  Slot s stages c_{i,l} omega_k =
// lam_i' (Psi_l Omega)_{:,k} of every row of kinds 1-3 (rows[q].coff: (h + 1) r doubles [l][k]) from k_narr_rot's records;
// thread tl evaluates simulation sim = y NR_SIMT + tl < n_sim on e_{k,tau} ~ N(0, 1) (RNG_NARR, rep = the model id):
//   kind 0: s e_{j,t} > 0;  kind 3: s H > 0;  kinds 1, 2: the share rule of nr_share, with H_{i,k} = sum_l (c_{i,l} omega_k) e_{k,t+h-l}.
// The CTA's count of simulations that satisfy every row is added to nok[s] (integers: the sum does not depend on the order).
// An empty slot or a failed model (sst != 0) adds nothing.
__global__ void k_narr_omega(const double* __restrict__ Lam, const double* __restrict__ rec, const nr_row* __restrict__ rows,
                             const int* __restrict__ sst, const unsigned long long* __restrict__ ids, int N, int r, int H, int nN, int nC,
                             int nP, int n_sim, int n_keep, unsigned long long seed, unsigned long long* __restrict__ nok) {
  DFM_SMEM(sm);
  const int s = DFM_BX, b = s / n_keep;
  if (sst[s] != 0) return;
  double* sCw = sm;
  int* cnt = (int*)(sCw + nC);
  const double* Lb = Lam + (size_t)b * N * r;
  const double* Ro = rec + (size_t)s * r * r * H;
  for (int q = 0; q < nN; ++q) {
    const nr_row w = rows[q];
    if (w.kind == 0) continue;
    for (int e = DFM_TID; e < (w.h + 1) * r; e += DFM_NT) {
      const int l = e / r, k = e % r;
      const double* pk = Ro + ((size_t)k * H + l) * r;
      double v = 0.0;
      for (int a = 0; a < r; ++a) v += Lb[w.series + (size_t)N * a] * pk[a];
      sCw[w.coff + e] = v;
    }
  }
  if (DFM_TID == 0) *cnt = 0;
  DFM_SYNC();
  const unsigned long long id = ids[b];
  int n = 0;
  for (int tl = DFM_TID; tl < NR_SIMT; tl += DFM_NT) {
    const long long sim = (long long)DFM_BY * NR_SIMT + tl;
    if (sim >= n_sim) continue;
    const unsigned long long e0 = (unsigned long long)sim * nP;
    bool ok = true;
    for (int q = 0; q < nN && ok; ++q) {
      const nr_row w = rows[q];
      if (w.kind == 0) {
        ok = w.sign * rng_normal(seed, id, RNG_NARR, (e0 + w.pos) * r + w.shock) > 0.0;
        continue;
      }
      const double* cw = sCw + w.coff;
      double hj = 0.0, mx = 0.0, sum = 0.0;
      for (int k = 0; k < r; ++k) {
        if (w.kind == 3 && k != w.shock) continue;
        double v = 0.0;
        for (int l = 0; l <= w.h; ++l)
          v = fma(cw[(size_t)l * r + k], rng_normal(seed, id, RNG_NARR, (e0 + w.pos + w.h - l) * r + k), v);
        if (w.kind == 3) { hj = w.sign * v; continue; }
        v = fabs(v);
        if (k == w.shock) hj = v;
        else { mx = v > mx ? v : mx; sum += v; }
      }
      ok = w.kind == 3 ? hj > 0.0 : (w.kind == 1 ? hj > mx : hj > sum);
    }
    n += ok;
  }
  if (n) atomicAdd(cnt, n);
  DFM_SYNC();
  if (DFM_TID == 0 && *cnt) atomicAdd(nok + s, (unsigned long long)*cnt);
}

// grid (ceil(S / NR_PT)), NR_PT threads.  weight[s] = n_sim / nok[s]; +Inf when nok = 0; NaN for an empty slot or a failed
// model.  n_ok, weight: S each, either may be NULL.
__global__ void k_narr_weight(const unsigned long long* __restrict__ nok, const int* __restrict__ sst, int S, int n_sim,
                              long long* __restrict__ n_ok, double* __restrict__ weight) {
  for (int tl = DFM_TID; tl < NR_PT; tl += DFM_NT) {
    const int s = DFM_BX * NR_PT + tl;
    if (s >= S) continue;
    const unsigned long long n = nok[s];
    if (n_ok) n_ok[s] = sst[s] != 0 ? 0 : (long long)n;
    if (weight) weight[s] = sst[s] != 0 ? DFM_NAN : (n ? (double)n_sim / (double)n : HUGE_VAL);
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Weighted percentiles over the replication axis, over the counted records (x not NaN, 0 < w < Inf): per quantile q, the first
// record i in sorted order with 100 sum_{j <= i} w_j >= q sum_j w_j in exact arithmetic (numpy's inverted_cdf rule with weights,
// without its rounding of the cumulative weights and of q / 100; with equal weights, numpy's unweighted inverted_cdf).
// recs: [n][d] row-major, w: [n]; grid = d statistics, NR_PT threads, shared npad + 2 (NR_PT + 1) doubles + 1 int + npad ints.  One bitonic sort of the (value,
// record index) pairs per statistic (records not counted sort last); the sorted values are then replaced by the weights
// w[index], summed in NR_PT chunks (in both builds) as double-double sums, and the chunk totals prefix-summed the same way.  Per
// quantile a binary search over the chunk prefixes and a walk through one chunk find i; the test of 100 times a prefix against q
// times the total is the exact sign of a sum of eight doubles.  The sums are exact while every partial sum fits in 106 bits of the
// smallest weight's grid (n <= 16 384 and max w / min w <= 2^36, so every narrative weight n_sim / n_ok).  out: [nq][d].
__device__ __forceinline__ bool wp_gt(double a, double b) { return is_nan(a) ? !is_nan(b) : (!is_nan(b) && a > b); }

__host__ __device__ inline size_t wpercentiles_smem_bytes(long long npad) {
  return (size_t)(npad + 2 * (NR_PT + 1) + 1) * 8 + (size_t)npad * 4;
}

// s + e = a + b exactly (Knuth's TwoSum)
__device__ __forceinline__ void wp_two_sum(double a, double b, double& s, double& e) {
  s = a + b;
  const double z = s - a;
  e = (a - (s - z)) + (b - z);
}

// (s, e) += w, renormalised so that |e| <= ulp(s) / 2: exact while s + e + w fits in 106 bits of the weights' grid
__device__ __forceinline__ void wp_dd_add(double& s, double& e, double w) {
  double t, err;
  wp_two_sum(s, w, t, err);
  err += e;
  s = t + err;
  e = err - (s - t);
}

// the rounded product, kept out of fma contraction (the TwoSums below need the product they are given)
__device__ __forceinline__ double wp_mul(double a, double b) {
#ifdef DFM_EMU
  return a * b;
#else
  return __dmul_rn(a, b);
#endif
}

// 100 (s + e) >= q (th + tl), exactly (0 <= q <= 100, 0 < s + e <= th + tl, |e| and |tl| about half an ulp of s and th):
// a1 - p1 = fl(100 s) - fl(q th) is within 2^-50 (100 th) of the difference, so its sign decides unless it is smaller than
// 2^-46 (100 th); then the four products split by fma and the sign of the eight-term sum from Shewchuk's grow-expansion (a
// non-overlapping expansion has the sign of its most significant non-zero component)
__device__ __forceinline__ bool wp_ge(double s, double e, double q, double th, double tl) {
  const double a1 = wp_mul(100.0, s), p1 = wp_mul(q, th);
  const double d = a1 - p1;
  if (fabs(d) > 0x1p-46 * (100.0 * th)) return d > 0.0;
  const double a2 = wp_mul(100.0, e), p2 = wp_mul(q, tl);
  const double x[8] = {a1, fma(100.0, s, -a1), a2, fma(100.0, e, -a2), -p1, -fma(q, th, -p1), -p2, -fma(q, tl, -p2)};
  double g[8];
#pragma unroll
  for (int a = 0; a < 8; ++a) {
    double Q = x[a];
#pragma unroll
    for (int b = 0; b < a; ++b) { double t, err; wp_two_sum(Q, g[b], t, err); g[b] = err; Q = t; }
    g[a] = Q;
  }
#pragma unroll
  for (int b = 7; b >= 0; --b) if (g[b] != 0.0) return g[b] > 0.0;
  return true;
}

__global__ void k_wpercentiles(const double* __restrict__ recs, const double* __restrict__ w, int n, int d, const double* __restrict__ q,
                               int nq, int npad, double* __restrict__ out) {
  DFM_SMEM(v);
  const int e = DFM_BX;
  double* ph = v + npad;                               // [NR_PT + 1] chunk prefixes (exclusive; ph[NR_PT] the total), high parts
  double* pl = ph + NR_PT + 1;                         //                                                                 low parts
  int* cnt = (int*)(pl + NR_PT + 1);
  int* ix = cnt + 2;
  if (DFM_TID == 0) *cnt = 0;
  DFM_SYNC();
  int c = 0;
  for (int i = DFM_TID; i < npad; i += DFM_NT) {
    double x = i < n ? recs[(size_t)i * d + e] : DFM_NAN;
    const double y = i < n ? w[i] : 0.0;
    if (is_nan(x) || !(y > 0.0 && y < HUGE_VAL)) x = DFM_NAN; else ++c;
    v[i] = x; ix[i] = i;
  }
  if (c) atomicAdd(cnt, c);
  DFM_SYNC();
#ifdef DFM_EMU
  for (int i = 1; i < npad; ++i) {
    const double x = v[i];
    const int y = ix[i];
    int j = i - 1;
    while (j >= 0 && wp_gt(v[j], x)) { v[j + 1] = v[j]; ix[j + 1] = ix[j]; --j; }
    v[j + 1] = x; ix[j + 1] = y;
  }
#else
  for (int k = 2; k <= npad; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < npad; i += blockDim.x) {
        const int l = i ^ j;
        if (l > i) {
          const double a = v[i], b = v[l];
          const bool up = (i & k) == 0;
          if (wp_gt(a, b) == up) { v[i] = b; v[l] = a; const int t = ix[i]; ix[i] = ix[l]; ix[l] = t; }
        }
      }
      __syncthreads();
    }
#endif
  const int m = *cnt;
  double* ww = v;                                      // (the values are read back from recs at the end)
  for (int i = DFM_TID; i < m; i += DFM_NT) ww[i] = w[ix[i]];
  DFM_SYNC();
  // chunk tl holds ww[tl ch .. (tl + 1) ch): its total, then the exclusive prefixes of the totals
  const int ch = (m + NR_PT - 1) / NR_PT;
  for (int tl = DFM_TID; tl < NR_PT; tl += DFM_NT) {
    double s = 0.0, el = 0.0;
    for (int i = tl * ch; i < m && i < (tl + 1) * ch; ++i) wp_dd_add(s, el, ww[i]);
    ph[tl + 1] = s; pl[tl + 1] = el;
  }
  DFM_SYNC();
  if (DFM_TID == 0) {
    double s = 0.0, el = 0.0;
    for (int tl = 0; tl < NR_PT; ++tl) {
      const double xh = ph[tl + 1], xl = pl[tl + 1];
      ph[tl] = s; pl[tl] = el;
      wp_dd_add(s, el, xh);
      wp_dd_add(s, el, xl);
    }
    ph[NR_PT] = s; pl[NR_PT] = el;
  }
  DFM_SYNC();
  for (int k = DFM_TID; k < nq; k += DFM_NT) {
    double r_ = DFM_NAN;
    if (m > 0) {
      const double qk = q[k], th = ph[NR_PT], tl_ = pl[NR_PT];
      int lo = 0, hi = NR_PT - 1;                      // the first chunk whose inclusive prefix reaches the threshold
      while (lo < hi) { const int mid = (lo + hi) >> 1; if (wp_ge(ph[mid + 1], pl[mid + 1], qk, th, tl_)) hi = mid; else lo = mid + 1; }
      double s = ph[lo], el = pl[lo];
      const int end = m < (lo + 1) * ch ? m : (lo + 1) * ch;
      int i = lo * ch < end ? lo * ch : end - 1;
      for (;; ++i) {                                   // (the chunk's last record reaches it: the loop ends inside the chunk)
        wp_dd_add(s, el, ww[i]);
        if (i >= end - 1 || wp_ge(s, el, qk, th, tl_)) break;
      }
      r_ = recs[(size_t)ix[i] * d + e];
    }
    out[(size_t)k * d + e] = r_;
  }
}

}  // namespace dfm
