// dfm_kernels_emb.cuh -- multi-CTA contraction kernels of the GENERAL state-space EM path for BALANCED panels (no NaN
// among the series in the model), any N, T, r <= 32, any p.  They replace k_em_contract_bal / k_em_mstep_series / the W, C
// loops of k_em_prep when one panel is too large for one CTA per phase (C3: N = 2000, r = 20, T = 2000, B = 1): both
// panel passes are split over the whole GPU --
//   E contraction  b_t = W'x_t, q_t = x_t'R^-1 x_t :  grid (64-period tiles, series splits, panels)
//   M contraction  S_xf = X'E[f],  S_xx            :  grid (64-series tiles, period splits, panels)
// on the FP64 tensor path (mma.sync.m8n8k4.f64 -> DMMA.8x8x4), fragments loaded straight from global / L2 (the panel of
// C3 is 32 MB: L2 resident across iterations; every 32-byte sector a fragment load touches is used completely).
// Partial results of the splits are combined by the LAST CTA to arrive (threadfence + counter), always in split order, so
// the result does not depend on the arrival order.  The last CTA of the M contraction also does the series' M-step
// (Lam_i = S_ff^-1 S_xf,i, R_i, W_i = Lam_i / R_i, log R_i) and its tile's share of C = Lam'R^-1 Lam.
// Spec: oracle/kalman_em.py (no reference code exists for the state-space EM, SURVEY.md 8 a').
#pragma once
#include "dfm_kernels_em.cuh"

namespace dfm {

#define EMB_TILE 64            // periods (E) / series (M) per CTA: 8 warps x one 8-row DMMA block
#define EMB_MAXSPLIT 256       // series (E) per split: bound of the shared-memory W stage

#ifndef DFM_EMU
#define EMB_DMMA(d_, a_, b_) asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n" : "+d"((d_)[0]), "+d"((d_)[1]) : "d"(a_), "d"(b_))
#define EMB_FENCE() __threadfence()
#else
#define EMB_FENCE() ((void)0)
#endif

__host__ __device__ inline int emb_pad(int x) { return x + ((4 - x % 16) + 16) % 16; }     // leading dimension == 4 (mod 16)

// E contraction.  grid (ceil(T/64), nsplit * B), 256 threads.  Shared: NCB*8*emb_pad(nper) + nper + 48 doubles.
// Bpart [nsplit][B][T x r], qpart [nsplit][B][T]; counters [B][ceil(T/64)] zero on entry (and on exit).
template <int NCB>
__global__ void k_emb_contract(const double* __restrict__ Xall, const double* __restrict__ Wall, const double* __restrict__ Rall,
                               const double* __restrict__ logRall, int T, int N, int r, int nsplit, int nper, int Bn,
                               double* __restrict__ Bpart, double* __restrict__ qpart, int* __restrict__ counters,
                               double* __restrict__ Bt_, double* __restrict__ qt_, double* __restrict__ slr_, int* __restrict__ nt_,
                               const EmState* st) {
  DFM_SMEM(sm);
  const int tile = DFM_BX, s = DFM_BY % nsplit, b = DFM_BY / nsplit;
  if (st[b].done || st[b].has_missing) return;
  const int ntiles = DFM_GX, npp = emb_pad(nper);
  double* Ws = sm;                         // [NCB*8][npp]   component-major, 0 for excluded series / components >= r
  double* rinv = Ws + (size_t)NCB * 8 * npp;  // [nper]      0 for excluded series
  double* red = rinv + nper;               // 48
  const double* X = Xall + (size_t)b * T * N; const double* W = Wall + (size_t)b * N * r; const double* R = Rall + (size_t)b * N;
  const int n0 = s * nper, n1 = (n0 + nper < N) ? n0 + nper : N;
  for (int e = DFM_TID; e < NCB * 8 * nper; e += DFM_NT) {
    const int a = e / nper, il = e % nper, i = n0 + il;
    double v = 0.0;
    if (i < n1 && a < r) { v = W[i + (size_t)N * a]; if (is_nan(W[i])) v = 0.0; }
    Ws[(size_t)a * npp + il] = v;
  }
  for (int il = DFM_TID; il < nper; il += DFM_NT) { const int i = n0 + il; rinv[il] = (i < n1 && !is_nan(W[i])) ? 1.0 / R[i] : 0.0; }
  DFM_SYNC();
  double* Bp = Bpart + (size_t)(s * Bn + b) * T * r; double* qp = qpart + (size_t)(s * Bn + b) * T;
#ifndef DFM_EMU
  {
    const int lane = DFM_LANE, lr = lane >> 2, lc = lane & 3;
    const int t = tile * EMB_TILE + DFM_WARP * 8 + lr;
    const bool tok = t < T;
    double d[NCB][2];
#pragma unroll
    for (int cb = 0; cb < NCB; ++cb) { d[cb][0] = 0.0; d[cb][1] = 0.0; }
    double qa = 0.0;
    const double* xc = X + (tok ? t : 0);
    const int nl = n1 - n0;
#pragma unroll 4
    for (int il0 = 0; il0 < nl; il0 += 4) {
      const int il = il0 + lc;
      const double ri = (il < nl) ? rinv[il] : 0.0;
      double x = (tok && ri > 0.0) ? xc[(size_t)T * (n0 + il)] : 0.0;
      qa += x * x * ri;
#pragma unroll
      for (int cb = 0; cb < NCB; ++cb) {
        const double wv = (il < nl) ? Ws[(size_t)(cb * 8 + lr) * npp + il] : 0.0;
        EMB_DMMA(d[cb], x, wv);
      }
    }
    qa += __shfl_xor_sync(0xffffffffu, qa, 1); qa += __shfl_xor_sync(0xffffffffu, qa, 2);
    if (tok) {
#pragma unroll
      for (int cb = 0; cb < NCB; ++cb) {
        const int a = cb * 8 + 2 * lc;
        if (a < r) Bp[t + (size_t)T * a] = d[cb][0];
        if (a + 1 < r) Bp[t + (size_t)T * (a + 1)] = d[cb][1];
      }
      if (lc == 0) qp[t] = qa;
    }
  }
#else
  for (int tl = 0; tl < EMB_TILE; ++tl) {
    const int t = tile * EMB_TILE + tl;
    if (t >= T) break;
    double q = 0.0;
    for (int a = 0; a < r; ++a) Bp[t + (size_t)T * a] = 0.0;
    for (int i = n0; i < n1; ++i) {
      const double ri = rinv[i - n0];
      if (!(ri > 0.0)) continue;
      const double x = X[t + (size_t)T * i];
      q += x * x * ri;
      for (int a = 0; a < r; ++a) Bp[t + (size_t)T * a] += x * Ws[(size_t)a * npp + (i - n0)];
    }
    qp[t] = q;
  }
#endif
  // ---- the last split of this (tile, panel) to arrive combines the partial sums, in split order
  int* flag = (int*)(red + 40);
  EMB_FENCE();
  DFM_SYNC();
  if (DFM_TID == 0) { const int old = atomicAdd(&counters[b * ntiles + tile], 1); *flag = (old == nsplit - 1); }
  DFM_SYNC();
  if (!*flag) return;
  EMB_FENCE();
  double sl = 0.0, nn = 0.0;
  const double* logR = logRall + (size_t)b * N;
  for (int i = DFM_TID; i < N; i += DFM_NT) if (!is_nan(W[i])) { sl += logR[i]; nn += 1.0; }
  sl = block_sum(sl, red); nn = block_sum(nn, red);
  const int tbase = tile * EMB_TILE;
  for (int e = DFM_TID; e < EMB_TILE * (r + 1); e += DFM_NT) {
    const int tl = e % EMB_TILE, a = e / EMB_TILE, t = tbase + tl;
    if (t >= T) continue;
    double v = 0.0;
    if (a < r) {
      for (int s2 = 0; s2 < nsplit; ++s2) v += Bpart[((size_t)(s2 * Bn + b) * r + a) * T + t];
      Bt_[(size_t)b * T * r + t + (size_t)T * a] = v;
    } else {
      for (int s2 = 0; s2 < nsplit; ++s2) v += qpart[(size_t)(s2 * Bn + b) * T + t];
      qt_[(size_t)b * T + t] = v; slr_[(size_t)b * T + t] = sl; nt_[(size_t)b * T + t] = (int)nn;
    }
  }
  if (DFM_TID == 0) counters[b * ntiles + tile] = 0;
}

// R_i, W_i = Lam_i / R_i, log R_i of a restricted series i from its corrected loadings li[0..r) (S0: S_ff); li[r] = 1/R_i.
// The same arithmetic as the unrestricted thread-per-series loop of emb_mstep_body, which keeps its own inline copy so that
// the unrestricted kernel compiles exactly as before.
__device__ __forceinline__ void emb_series_finish(double* li, const double* sx, const double* S0, int r, int T, int N, int i, double* Lam,
                                                  double* R, double* W, double* logR, int* bad) {
  const double sxx = sx[r];
  double q1 = 0.0, q2 = 0.0;
  for (int a = 0; a < r; ++a) {
    q1 += li[a] * sx[a];
    double v = 0.0;
    for (int c = 0; c < r; ++c) v += S0[a + r * c] * li[c];
    q2 += li[a] * v;
  }
  const double Ri = (sxx - 2.0 * q1 + q2) / (double)T;
  R[i] = Ri;
  const double rinv = 1.0 / Ri;
  if (!(Ri > 0.0)) *bad = 1;
  for (int a = 0; a < r; ++a) { Lam[i + (size_t)N * a] = li[a]; W[i + (size_t)N * a] = li[a] * rinv; }
  logR[i] = log(Ri);
  li[r] = rinv;
}

// M contraction + measurement M-step.  grid (ceil(N/64), tsplit * B), 256 threads.
// Shared: 2 r*r + 2 * 64*(r+1) + 96 doubles (+ em_constr_scratch(r) when CON).  Spart [tsplit][B][N x r], sxxpart [tsplit][B][N];
// counters [B][ceil(N/64)].  Cpart [B][ceil(N/64)][r x r]: this tile's share of C = Lam' R^-1 Lam (summed by k_emb_close).
// k_emb_mstep_constr (the call has restrictions on the loadings, CON): the thread-per-series loop leaves the restricted series
// of the tile at Lam_i = S_ff^-1 S_xf,i; thread 0 then corrects them one by one (lam_constr_correct with the shared Cholesky
// factor of S_ff, scratch in shared memory) before their R_i, W_i, log R_i and the tile's share of C are formed.  Both
// kernels are the one body below; without CON it compiles to the unrestricted kernel alone.
template <int NCB, bool CON>
__device__ __forceinline__ void emb_mstep_body(const double* __restrict__ Xall, const double* __restrict__ Fs_,
                                               const double* __restrict__ SffAll_, int T, int N, int r, int tsplit, int tper, int Bn,
                                               double* __restrict__ Spart, double* __restrict__ sxxpart, int* __restrict__ counters,
                                               double* __restrict__ LamAll, double* __restrict__ Rall, double* __restrict__ Wall,
                                               double* __restrict__ logRall, double* __restrict__ Cpart, EmState* st, EmConstr cs) {
  DFM_SMEM(sm);
  const int tile = DFM_BX, s = DFM_BY % tsplit, b = DFM_BY / tsplit;
  if (st[b].done || st[b].has_missing) return;
  const int ntiles = DFM_GX;
  const double* X = Xall + (size_t)b * T * N; const double* Fs = Fs_ + (size_t)b * T * r;
  double* Lam = LamAll + (size_t)b * N * r; double* R = Rall + (size_t)b * N;
  const int ta = s * tper, tb = (ta + tper < T) ? ta + tper : T;
  double* Sp = Spart + (size_t)(s * Bn + b) * N * r; double* xp = sxxpart + (size_t)(s * Bn + b) * N;
#ifndef DFM_EMU
  {
    const int lane = DFM_LANE, lr = lane >> 2, lc = lane & 3;
    const int i = tile * EMB_TILE + DFM_WARP * 8 + lr;
    const bool iok = i < N && !is_nan(Lam[i < N ? i : 0]);
    double d[NCB][2];
#pragma unroll
    for (int cb = 0; cb < NCB; ++cb) { d[cb][0] = 0.0; d[cb][1] = 0.0; }
    double sx = 0.0;
    const double* xr = X + (size_t)T * (iok ? i : 0);
#pragma unroll 4
    for (int t0 = ta; t0 < tb; t0 += 4) {
      const int t = t0 + lc;
      const bool tk = t < tb;
      const double x = (iok && tk) ? xr[t] : 0.0;
      sx += x * x;
#pragma unroll
      for (int cb = 0; cb < NCB; ++cb) {
        const int a = cb * 8 + lr;
        const double f = (tk && a < r) ? Fs[t + (size_t)T * a] : 0.0;
        EMB_DMMA(d[cb], x, f);
      }
    }
    sx += __shfl_xor_sync(0xffffffffu, sx, 1); sx += __shfl_xor_sync(0xffffffffu, sx, 2);
    if (i < N) {
#pragma unroll
      for (int cb = 0; cb < NCB; ++cb) {
        const int a = cb * 8 + 2 * lc;
        if (a < r) Sp[i + (size_t)N * a] = d[cb][0];
        if (a + 1 < r) Sp[i + (size_t)N * (a + 1)] = d[cb][1];
      }
      if (lc == 0) xp[i] = sx;
    }
  }
#else
  for (int il = 0; il < EMB_TILE; ++il) {
    const int i = tile * EMB_TILE + il;
    if (i >= N) break;
    const bool iok = !is_nan(Lam[i]);
    double sx = 0.0;
    for (int a = 0; a < r; ++a) Sp[i + (size_t)N * a] = 0.0;
    if (iok) for (int t = ta; t < tb; ++t) {
      const double x = X[t + (size_t)T * i];
      sx += x * x;
      for (int a = 0; a < r; ++a) Sp[i + (size_t)N * a] += x * Fs[t + (size_t)T * a];
    }
    xp[i] = sx;
  }
#endif
  double* S = sm;                          // r x r: S_ff, then its Cholesky factor
  double* S0 = S + r * r;                  // r x r: S_ff
  double* lamt = S0 + r * r;               // [64][r+1]: lam_i, 1/R_i (0 = excluded)
  double* red = lamt + EMB_TILE * (r + 1); // 48
  int* flag = (int*)(red + 40);
  EMB_FENCE();
  DFM_SYNC();
  if (DFM_TID == 0) { const int old = atomicAdd(&counters[b * ntiles + tile], 1); flag[0] = (old == tsplit - 1); flag[1] = 0; }
  DFM_SYNC();
  if (!flag[0]) return;
  EMB_FENCE();
  for (int e = DFM_TID; e < r * r; e += DFM_NT) { S[e] = SffAll_[(size_t)b * r * r + e]; S0[e] = S[e]; }
  DFM_SYNC();
  bm_chol(S, r, r, &flag[1]);
  // split partials -> shared memory (all threads, independent loads), then one thread per series for the r x r solve
  double* sxf = lamt + EMB_TILE * (r + 1) + 48;          // [64][r + 1]: S_xf,i and S_xx,i
  for (int e = DFM_TID; e < EMB_TILE * (r + 1); e += DFM_NT) {
    const int il = e % EMB_TILE, a = e / EMB_TILE, i = tile * EMB_TILE + il;
    double v = 0.0;
    if (i < N) {
      if (a < r) { for (int s2 = 0; s2 < tsplit; ++s2) v += Spart[((size_t)(s2 * Bn + b) * r + a) * N + i]; }
      else for (int s2 = 0; s2 < tsplit; ++s2) v += sxxpart[(size_t)(s2 * Bn + b) * N + i];
    }
    sxf[(size_t)il * (r + 1) + a] = v;
  }
  DFM_SYNC();
  for (int il = DFM_TID; il < EMB_TILE; il += DFM_NT) {
    const int i = tile * EMB_TILE + il;
    double* li = lamt + (size_t)il * (r + 1);
    const double* sx = sxf + (size_t)il * (r + 1);
    for (int a = 0; a <= r; ++a) li[a] = 0.0;
    if (i >= N || is_nan(Lam[i]) || is_nan(R[i])) continue;
    const double sxx = sx[r];
    for (int a = 0; a < r; ++a) li[a] = sx[a];
    double q1 = 0.0, q2 = 0.0;
    // L y = sxf ; L' lam = y   (y and lam overwrite li)
    for (int a = 0; a < r; ++a) { double v = li[a]; for (int c = 0; c < a; ++c) v -= S[a + r * c] * li[c]; li[a] = v / S[a + r * a]; }
    for (int a = r - 1; a >= 0; --a) { double v = li[a]; for (int c = a + 1; c < r; ++c) v -= S[c + r * a] * li[c]; li[a] = v / S[a + r * a]; }
    if constexpr (CON) { if (cs.off[i + 1] > cs.off[i]) continue; }     // restricted: corrected and finished below
    for (int a = 0; a < r; ++a) {
      q1 += li[a] * sx[a];
      double v = 0.0;
      for (int c = 0; c < r; ++c) v += S0[a + r * c] * li[c];
      q2 += li[a] * v;
    }
    const double Ri = (sxx - 2.0 * q1 + q2) / (double)T;
    R[i] = Ri;
    const double rinv = 1.0 / Ri;
    if (!(Ri > 0.0)) flag[1] = 1;
    for (int a = 0; a < r; ++a) { Lam[i + (size_t)N * a] = li[a]; Wall[(size_t)b * N * r + i + (size_t)N * a] = li[a] * rinv; }
    logRall[(size_t)b * N + i] = log(Ri);
    li[r] = rinv;
  }
  DFM_SYNC();
  if constexpr (CON) if (DFM_TID == 0) {
    double* ws = sxf + (size_t)EMB_TILE * (r + 1);
    for (int il = 0; il < EMB_TILE; ++il) {
      const int i = tile * EMB_TILE + il;
      if (i >= N) break;
      const int q0 = cs.off[i], m = cs.off[i + 1] - q0;
      if (m == 0 || is_nan(Lam[i]) || is_nan(R[i])) continue;
      double* li = lamt + (size_t)il * (r + 1);
      if (lam_constr_correct(li, r, cs.H + (size_t)q0 * r, cs.h + q0, m, ws, [&](double* v) {
            for (int a = 0; a < r; ++a) { double u = v[a]; for (int c = 0; c < a; ++c) u -= S[a + r * c] * v[c]; v[a] = u / S[a + r * a]; }
            for (int a = r - 1; a >= 0; --a) { double u = v[a]; for (int c = a + 1; c < r; ++c) u -= S[c + r * a] * v[c]; v[a] = u / S[a + r * a]; }
          })) flag[1] = 1;
      emb_series_finish(li, sxf + (size_t)il * (r + 1), S0, r, T, N, i, Lam, R, Wall + (size_t)b * N * r, logRall + (size_t)b * N, &flag[1]);
    }
  }
  if constexpr (CON) DFM_SYNC();
  for (int e = DFM_TID; e < r * r; e += DFM_NT) {
    const int a = e % r, c = e / r;
    double v = 0.0;
    for (int il = 0; il < EMB_TILE; ++il) { const double* li = lamt + (size_t)il * (r + 1); v += li[a] * li[r] * li[c]; }
    Cpart[((size_t)b * ntiles + tile) * r * r + e] = v;
  }
  if (DFM_TID == 0) { counters[b * ntiles + tile] = 0; if (flag[1]) st[b].status = 3; }
}

template <int NCB>
__global__ void k_emb_mstep(const double* __restrict__ Xall, const double* __restrict__ Fs_, const double* __restrict__ SffAll_,
                            int T, int N, int r, int tsplit, int tper, int Bn, double* __restrict__ Spart,
                            double* __restrict__ sxxpart, int* __restrict__ counters, double* __restrict__ LamAll,
                            double* __restrict__ Rall, double* __restrict__ Wall, double* __restrict__ logRall,
                            double* __restrict__ Cpart, EmState* st) {
  emb_mstep_body<NCB, false>(Xall, Fs_, SffAll_, T, N, r, tsplit, tper, Bn, Spart, sxxpart, counters, LamAll, Rall, Wall, logRall,
                             Cpart, st, EmConstr{nullptr, nullptr, nullptr});
}

template <int NCB>
__global__ void k_emb_mstep_constr(const double* __restrict__ Xall, const double* __restrict__ Fs_, const double* __restrict__ SffAll_,
                                   int T, int N, int r, int tsplit, int tper, int Bn, double* __restrict__ Spart,
                                   double* __restrict__ sxxpart, int* __restrict__ counters, double* __restrict__ LamAll,
                                   double* __restrict__ Rall, double* __restrict__ Wall, double* __restrict__ logRall,
                                   double* __restrict__ Cpart, EmState* st, EmConstr cs) {
  emb_mstep_body<NCB, true>(Xall, Fs_, SffAll_, T, N, r, tsplit, tper, Bn, Spart, sxxpart, counters, LamAll, Rall, Wall, logRall,
                            Cpart, st, cs);
}

// Closing step of an iteration on the balanced multi-CTA path: commit the transition M-step, iteration count /
// convergence (as k_em_prep does), and C = sum of the tiles' shares.  grid (B), 128 threads.
__global__ void k_emb_close(int N, int r, int p, int ntilesM, const double* __restrict__ Cpart, double* __restrict__ Call,
                            double* __restrict__ A, const double* __restrict__ Anew, double* __restrict__ Q,
                            const double* __restrict__ Qnew, EmState* st, int max_iter, int commit) {
  const int b = DFM_BX;
  if (st[b].done || st[b].has_missing) return;
  const int rk = r * r * p, rr = r * r;
  if (commit) {
    for (int e = DFM_TID; e < rk; e += DFM_NT) A[(size_t)b * rk + e] = Anew[(size_t)b * rk + e];
    for (int e = DFM_TID; e < rr; e += DFM_NT) Q[(size_t)b * rr + e] = Qnew[(size_t)b * rr + e];
  }
  for (int e = DFM_TID; e < rr; e += DFM_NT) {
    double v = 0.0;
    for (int tl = 0; tl < ntilesM; ++tl) v += Cpart[((size_t)b * ntilesM + tl) * rr + e];
    Call[(size_t)b * rr + e] = v;
  }
  DFM_SYNC();
  for (int e = DFM_TID; e < rr; e += DFM_NT) {             // exact symmetry, as the a >= c loop of k_em_prep gives
    const int a = e % r, c = e / r;
    if (a > c) Call[(size_t)b * rr + c + r * a] = Call[(size_t)b * rr + a + r * c];
  }
  if (DFM_TID == 0 && commit) {
    st[b].iters += 1;
    if (st[b].conv_pending || st[b].iters >= max_iter || st[b].status == 3) st[b].done = 1;
  }
}

// C = Lam' R^-1 Lam of the INITIAL parameters, tile by tile (the iterations get it from k_emb_mstep).  grid (ceil(N/64), B).
__global__ void k_emb_cinit(const double* __restrict__ LamAll, const double* __restrict__ Wall, int N, int r,
                            double* __restrict__ Cpart, const EmState* st) {
  const int tile = DFM_BX, b = DFM_BY, ntiles = DFM_GX;
  if (st[b].done || st[b].has_missing) return;
  const double* Lam = LamAll + (size_t)b * N * r; const double* W = Wall + (size_t)b * N * r;
  const int i0 = tile * EMB_TILE, i1 = (i0 + EMB_TILE < N) ? i0 + EMB_TILE : N;
  for (int e = DFM_TID; e < r * r; e += DFM_NT) {
    const int a = e % r, c = e / r;
    double v = 0.0;
    for (int i = i0; i < i1; ++i) { const double w = W[i + (size_t)N * a]; if (!is_nan(w)) v += w * Lam[i + (size_t)N * c]; }
    Cpart[((size_t)b * ntiles + tile) * r * r + e] = v;
  }
}

// EM initialisation on the same machinery: per-panel flags (any NaN in the panel?) -> EmState.has_missing / an int copy.
__global__ void k_emb_init_flags(const double* __restrict__ Xall, int T, int N, EmState* st, int* __restrict__ miss) {
  const int i = DFM_BX, b = DFM_BY;
  const double* x = Xall + ((size_t)b * N + i) * T;
  int bad = 0;
  for (int t = DFM_TID; t < T; t += DFM_NT) if (is_nan(x[t])) bad = 1;
  if (bad) { st[b].has_missing = 1; miss[b] = 1; }       // benign race: all writers store 1
}

}  // namespace dfm
