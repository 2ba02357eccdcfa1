// dfm_kernels_sign.cuh -- shocks identified by sign restrictions on series responses, many models at once
// (dfm_sign_restrictions).  Per model (Lam, R, A, Q), L = chol(Q), Psi_h = [M^h]_{1:r,1:r} L and c_{i,h} = lam_i' Psi_h; a
// candidate rotation Omega = Q_Z diag(sign(diag R_Z)) of an r x r standard normal Z is kept when every restricted shock's rows
// rho = (i, h, j, s) give s c_{i,h} omega_j of one strict sign (include/dfm_b200.h has the definition):
//   k_sr_prep, k_irf  (dfm_kernels_resp.cuh, dfm_kernels_np.cuh) Psi_h of every model
//   k_sign_prep       one CTA per model: the rows' s c_{i,h}, the model's status, the pick state reset
//   k_sign_cand       one thread per candidate: draws Z column by column, Gram-Schmidt, tests the rows of each restricted shock
//                     and stops at the first failing one; one accept bit per candidate
//   k_sign_pick       one CTA per model: ordered scan of the accept bits -> the accept count and the first n_keep ids
//   k_sign_rot        one CTA per kept slot: rebuilds the candidate's columns with k_sign_cand's routine (the same bits), the
//                     flips, the rest of Omega, and the records Psi_h Omega in k_irf's layout for k_series_resp
// Gram-Schmidt with positive normalisation gives Q_Z diag(sign(diag R_Z)) directly, and column j depends on Z's columns 0..j
// only, so a rejected candidate never draws the columns after the failing shock.  Explicit fma in the column routine keeps
// k_sign_cand and k_sign_rot on the same roundings.  The spec is tests/sign_oracle.py.
#pragma once
#include "dfm_common.cuh"
#include "dfm_kernels_rep.cuh"

namespace dfm {

enum { RNG_SIGN = 18 };        // Z[a, j] of candidate c: element c r^2 + a + r j

#define SG_NT 64               // candidates (threads) per CTA of k_sign_cand: two 32-candidate tiles
#define SG_TILE 32             // candidates per accept word
#define SG_PT 256              // threads of k_sign_pick
#define SG_PW 4                // accept words per k_sign_pick thread and round
#define SG_RMAX 16             // r bound: the candidate columns live in shared memory
#define SG_NRMAX 256           // restriction rows bound: staged per CTA

__device__ __forceinline__ int sg_popc(unsigned v) {
#ifdef DFM_EMU
  return __builtin_popcount(v);
#else
  return __popc(v);
#endif
}

// The stream of one candidate's normals, consumed in increasing element order: each Philox block gives the pair (2m, 2m + 1),
// the second is kept for the next element (rng_normal's values).
struct sg_rng {
  unsigned long long seed, id, ec;
  double vc;
};
__device__ __forceinline__ double sg_normal(sg_rng& g, unsigned long long e) {
  if (e == g.ec) return g.vc;
  double u0, u1;
  rng_u2(g.seed, g.id, RNG_SIGN, e >> 1, u0, u1);
  const double rad = sqrt(-2.0 * log(u0)), ang = 6.283185307179586476925286766559 * u1;
  if (e & 1) return rad * sin(ang);
  g.ec = e + 1; g.vc = rad * sin(ang);
  return rad * cos(ang);
}

// Column j of Omega: Z's column j (elements e0 .. e0 + r - 1), orthogonalised against columns 0 .. j-1 by classical
// Gram-Schmidt with one re-orthogonalisation pass, normalised.  Column l, element a at Q[(l r + a) s]; W: r doubles of scratch
// at stride s.
__device__ __forceinline__ void sg_column(double* Q, double* W, int s, int r, int j, sg_rng& g, unsigned long long e0) {
  double* z = Q + (size_t)j * r * s;
  for (int a = 0; a < r; ++a) { const double v = sg_normal(g, e0 + a); z[(size_t)a * s] = v; W[(size_t)a * s] = v; }
  if (j > 0) {
    for (int l = 0; l < j; ++l) {                      // W = z - sum_l (q_l'z) q_l
      const double* q = Q + (size_t)l * r * s;
      double d = 0.0;
      for (int a = 0; a < r; ++a) d = fma(q[(size_t)a * s], z[(size_t)a * s], d);
      for (int a = 0; a < r; ++a) W[(size_t)a * s] = fma(-d, q[(size_t)a * s], W[(size_t)a * s]);
    }
    for (int a = 0; a < r; ++a) z[(size_t)a * s] = W[(size_t)a * s];
    for (int l = 0; l < j; ++l) {                      // z = W - sum_l (q_l'W) q_l
      const double* q = Q + (size_t)l * r * s;
      double d = 0.0;
      for (int a = 0; a < r; ++a) d = fma(q[(size_t)a * s], W[(size_t)a * s], d);
      for (int a = 0; a < r; ++a) z[(size_t)a * s] = fma(-d, q[(size_t)a * s], z[(size_t)a * s]);
    }
  }
  double n2 = 0.0;
  for (int a = 0; a < r; ++a) n2 = fma(z[(size_t)a * s], z[(size_t)a * s], n2);
  const double inv = 1.0 / sqrt(n2);
  for (int a = 0; a < r; ++a) z[(size_t)a * s] *= inv;
}

// +1: every row gives s c omega > 0;  -1: every row < 0 (the column is flipped);  0: rejected.  Cr: n rows of s c (r each).
__device__ __forceinline__ int sg_test(const double* Cr, int n, const double* w, int s, int r) {
  bool pos = true, neg = true;
  for (int q = 0; q < n && (pos || neg); ++q) {
    double v = 0.0;
    for (int a = 0; a < r; ++a) v = fma(Cr[(size_t)q * r + a], w[(size_t)a * s], v);
    pos = pos && v > 0.0;
    neg = neg && v < 0.0;
  }
  return pos ? 1 : (neg ? -1 : 0);
}

// grid (B), 64 threads, shared 8 bytes.  Lam N x r, R N per model; irf: k_irf's records ([b][j][h][a] = (Psi_h)_{a j});
// rows (series rs, horizon rh, sign sg) sorted by shock.  C[b][rho][a] = s_rho (lam_{i_rho}' Psi_{h_rho})_a.  st[b] (k_sr_prep's)
// becomes DFM_ERR_ARG when a restricted series is out of the model; the pick state (nacc = 0, cand = -1) is reset.
__global__ void k_sign_prep(const double* __restrict__ Lam, const double* __restrict__ R, const double* __restrict__ irf, int N, int r,
                            int H, int nR, const int* __restrict__ rs, const int* __restrict__ rh, const int* __restrict__ sg, int n_keep,
                            int* __restrict__ st, double* __restrict__ C, long long* __restrict__ nacc, long long* __restrict__ cand) {
  DFM_SMEM(sm);
  int* flag = (int*)sm;
  const int b = DFM_BX;
  const double* Lb = Lam + (size_t)b * N * r;
  const double* P = irf + (size_t)b * r * r * H;
  if (DFM_TID == 0) {
    int out = 0;
    for (int q = 0; q < nR; ++q) {
      const int i = rs[q];
      bool bad = is_nan(R[(size_t)b * N + i]);
      for (int a = 0; a < r; ++a) bad = bad || is_nan(Lb[i + (size_t)N * a]);
      if (bad) out = 1;
    }
    *flag = out;
  }
  for (int e = DFM_TID; e < nR * r; e += DFM_NT) {
    const int q = e / r, a = e % r, i = rs[q];
    const double* pa = P + ((size_t)a * H + rh[q]) * r;          // (Psi_h)_{l a}, l = 0 .. r-1
    double c = 0.0;
    for (int l = 0; l < r; ++l) c += Lb[i + (size_t)N * l] * pa[l];
    C[((size_t)b * nR + q) * r + a] = sg[q] > 0 ? c : -c;
  }
  for (int e = DFM_TID; e < n_keep; e += DFM_NT) cand[(size_t)b * n_keep + e] = -1;
  DFM_SYNC();
  if (DFM_TID == 0) {
    nacc[b] = 0;
    if (st[b] == 0 && *flag) st[b] = DFM_ERR_ARG;
  }
}

// Shared memory of k_sign_cand: the candidates' columns 0 .. nj-1 and a scratch column (nj + 1) r SG_NT, the rows nR r, the
// per-shock row offsets.
__host__ __device__ inline size_t sign_cand_smem_bytes(int r, int nj, int nR) {
  return ((size_t)(nj + 1) * r * SG_NT + (size_t)nR * r) * 8 + (size_t)(nj + 1) * 4;
}

// grid (ntile / 2, B), SG_NT threads.  Candidates c0 + t, t < ntile SG_TILE, of model b (id ids[b]); those >= n_rot are
// rejected.  off: nj + 1 row offsets (shock j's rows are off[j] .. off[j+1]-1 of C, nj = the last restricted shock + 1).
// mask[b][w] bit l: candidate c0 + w SG_TILE + l accepted.  A model with st != 0 accepts nothing.
__global__ void k_sign_cand(const double* __restrict__ C, const int* __restrict__ off, const int* __restrict__ st, int r, int nR, int nj,
                            long long c0, long long n_rot, int ntile, unsigned long long seed, const unsigned long long* __restrict__ ids,
                            unsigned* __restrict__ mask) {
  DFM_SMEM(sm);
  const int b = DFM_BY;
  double* sQ = sm;                                     // [(l r + a)][SG_NT]  columns, then the scratch column
  double* sC = sQ + (size_t)(nj + 1) * r * SG_NT;      // [rho][a]
  int* sOff = (int*)(sC + (size_t)nR * r);
  for (int e = DFM_TID; e < nR * r; e += DFM_NT) sC[e] = C[(size_t)b * nR * r + e];
  for (int e = DFM_TID; e <= nj; e += DFM_NT) sOff[e] = off[e];
  DFM_SYNC();
  const bool bad = st[b] != 0;
  const unsigned long long id = ids[b], rr = (unsigned long long)r * r;
  for (int tl = DFM_TID; tl < SG_NT; tl += DFM_NT) {
    const long long c = c0 + (long long)DFM_BX * SG_NT + tl;
    bool ok = !bad && c < n_rot;
    if (ok) {
      sg_rng g{seed, id, ~0ull, 0.0};
      double* Q = sQ + tl;
      for (int j = 0; j < nj && ok; ++j) {
        sg_column(Q, Q + (size_t)nj * r * SG_NT, SG_NT, r, j, g, (unsigned long long)c * rr + (unsigned long long)r * j);
        ok = sg_test(sC + (size_t)sOff[j] * r, sOff[j + 1] - sOff[j], Q + (size_t)j * r * SG_NT, SG_NT, r) != 0;
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

// grid (B), SG_PT threads, shared 2 SG_PT ints.  Appends the accepted ids of one batch of k_sign_cand (ntile words per model
// from candidate c0) to cand[b] while fewer than n_keep are kept, in candidate order, and adds the batch's count to nacc[b].
// Per round every thread counts SG_PW consecutive words; an inclusive scan (Hillis-Steele, double-buffered) gives each thread
// the slot of its first id.
__global__ void k_sign_pick(const unsigned* __restrict__ mask, int ntile, long long c0, int n_keep, const int* __restrict__ st,
                            long long* __restrict__ nacc, long long* __restrict__ cand) {
  DFM_SMEM(sm);
  const int b = DFM_BX;
  if (st[b] != 0) return;
  int* A = (int*)sm;
  int* B = A + SG_PT;
  const unsigned* mb = mask + (size_t)b * ntile;
  long long* cb = cand + (size_t)b * n_keep;
  long long run = nacc[b];
  for (int w0 = 0; w0 < ntile; w0 += SG_PT * SG_PW) {
    for (int tl = DFM_TID; tl < SG_PT; tl += DFM_NT) {
      int n = 0;
      for (int q = 0; q < SG_PW; ++q) { const int w = w0 + tl * SG_PW + q; if (w < ntile) n += sg_popc(mb[w]); }
      A[tl] = n;
    }
    DFM_SYNC();
    int *in = A, *out = B;
    for (int o = 1; o < SG_PT; o <<= 1) {
      for (int tl = DFM_TID; tl < SG_PT; tl += DFM_NT) out[tl] = in[tl] + (tl >= o ? in[tl - o] : 0);
      DFM_SYNC();
      int* t = in; in = out; out = t;
    }
    if (run < n_keep)
      for (int tl = DFM_TID; tl < SG_PT; tl += DFM_NT) {
        long long k = run + (tl ? in[tl - 1] : 0);
        for (int q = 0; q < SG_PW && k < n_keep; ++q) {
          const int w = w0 + tl * SG_PW + q;
          if (w >= ntile) break;
          for (unsigned m = mb[w]; m && k < n_keep; m &= m - 1) {
            const int l = sg_popc((m & (0u - m)) - 1u);      // (the lowest set bit)
            cb[k++] = c0 + (long long)w * SG_TILE + l;
          }
        }
      }
    run += in[SG_PT - 1];
    DFM_SYNC();                                        // (A and B are rewritten by the next round)
  }
  if (DFM_TID == 0) nacc[b] = run;
}

// Shared memory of k_sign_rot: Omega and a scratch column (r + 1) r, the rows nR r, the offsets, the flips.
__host__ __device__ inline size_t sign_rot_smem_bytes(int r, int nj, int nR) {
  return ((size_t)(r + 1) * r + (size_t)nR * r) * 8 + (size_t)(nj + 1 + r) * 4;
}

// grid (B n_keep), 64 threads.  Slot s of model b = s / n_keep holds candidate cand[s] (-1: empty).  Writes Omega (r x r,
// column-major; may be NULL), the records rec[s][j][h][a] = (Psi_h Omega)_{a j} of all r shocks (k_irf's layout, for
// k_series_resp), and sst[s] = 0, or 3 for an empty slot or a model with st != 0 (NaN Omega and records).
__global__ void k_sign_rot(const double* __restrict__ irf, const double* __restrict__ C, const int* __restrict__ off,
                           const int* __restrict__ st, const long long* __restrict__ cand, int r, int H, int nR, int nj, int n_keep,
                           unsigned long long seed, const unsigned long long* __restrict__ ids, double* __restrict__ rot,
                           double* __restrict__ rec, int* __restrict__ sst) {
  DFM_SMEM(sm);
  const int s = DFM_BX, b = s / n_keep;
  double* sQ = sm;                                     // [j][a] Omega, then the scratch column
  double* sC = sQ + (size_t)(r + 1) * r;
  int* sOff = (int*)(sC + (size_t)nR * r);
  int* flip = sOff + nj + 1;
  const long long c = cand[s];
  const bool bad = st[b] != 0 || c < 0;
  if (!bad) {
    for (int e = DFM_TID; e < nR * r; e += DFM_NT) sC[e] = C[(size_t)b * nR * r + e];
    for (int e = DFM_TID; e <= nj; e += DFM_NT) sOff[e] = off[e];
    DFM_SYNC();
    if (DFM_TID == 0) {
      sg_rng g{seed, ids[b], ~0ull, 0.0};
      const unsigned long long rr = (unsigned long long)r * r;
      for (int j = 0; j < r; ++j) {
        sg_column(sQ, sQ + (size_t)r * r, 1, r, j, g, (unsigned long long)c * rr + (unsigned long long)r * j);
        flip[j] = j < nj ? sg_test(sC + (size_t)sOff[j] * r, sOff[j + 1] - sOff[j], sQ + (size_t)j * r, 1, r) : 1;
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
  if (DFM_TID == 0) sst[s] = bad ? 3 : 0;
}

}  // namespace dfm
