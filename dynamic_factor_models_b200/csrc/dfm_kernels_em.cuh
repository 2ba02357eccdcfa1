// dfm_kernels_em.cuh -- GENERAL (any r, p with k = r*p <= 48, any N, T, missing data) kernels of the
// state-space EM, row a' of SURVEY.md section 8.  No reference code exists for this path
// (dfm_functions.ipynb:23 is an empty placeholder); the spec is oracle/kalman_em.py.
// One EM iteration = contraction -> k_em_filter_smooth -> measurement M-step -> closing step:
//   panels with missing data:  k_em_contract (masked C_t) -> k_em_filter_smooth -> k_em_mstep_series -> k_em_prep
//   balanced panels (r <= 32):  k_emb_contract -> k_em_filter_smooth -> k_emb_mstep -> k_emb_close   (dfm_kernels_emb.cuh)
// k_em_filter_smooth (one CTA, or a thread-block cluster, per panel) holds the filter, the smoother and the transition
// M-step: explicit covariance steps, frozen steps, and frozen RUNS as parallel-in-time scans on the tensor path
// (em_run_scan_tc); the small dense helpers it uses (block-cooperative Cholesky, transposed solves, DMMA tile products)
// live in dfm_common.cuh.  The fused small-k fast path lives in dfm_kernels_fused*.cuh; this file is also the path the
// host-emulation tests exercise (DMMA loops have plain twins under DFM_EMU).
#pragma once
#include "dfm_common.cuh"

namespace dfm {

struct EmState {           // one per panel
  double ll, ll_prev;
  int iters, done, status, has_missing, conv_pending, pad;
};

#define DFM_LOG2PI 1.8378770664093454835606594728112

// any NaN among the series that are in the model?  grid (N, B)
__global__ void k_em_scan(const double* __restrict__ X, const double* __restrict__ Lam, int T, int N, int r, EmState* st) {
  int i = DFM_BX, b = DFM_BY;
  if (is_nan(Lam[(size_t)b * N * r + i])) return;     // excluded series
  const double* x = X + ((size_t)b * N + i) * T;
  int miss = 0;
  for (int t = DFM_TID; t < T; t += DFM_NT) if (is_nan(x[t])) miss = 1;
  if (miss) st[b].has_missing = 1;     // benign race: all writers store 1
}

__global__ void k_em_state_init(EmState* st) {
  if (DFM_TID != 0) return;
  int b = DFM_BX;
  st[b].ll = 0.0; st[b].ll_prev = 0.0; st[b].iters = 0; st[b].done = 0; st[b].status = 0;
  st[b].has_missing = 0; st[b].conv_pending = 0;
}

// Default prior P0 = sum_j M^j Qt M'^j by doubling (oracle lyapunov_doubling, 12 steps).
// grid (B), one block; shared 3*k*k doubles.
__global__ void k_lyapunov(const double* __restrict__ Aall, const double* __restrict__ Qall, int r, int p,
                           double* __restrict__ P0all, int steps) {
  DFM_SMEM(sm);
  int b = DFM_BX, k = r * p, kk = k * k;
  const double* A = Aall + (size_t)b * r * k; const double* Q = Qall + (size_t)b * r * r;
  double* P = sm; double* Mj = P + kk; double* T1 = Mj + kk;
  for (int e = DFM_TID; e < kk; e += DFM_NT) {
    int i = e % k, j = e / k;
    P[e] = (i < r && j < r) ? Q[i + r * j] : 0.0;
    Mj[e] = (i < r) ? A[i + r * j] : ((j == i - r) ? 1.0 : 0.0);
  }
  DFM_SYNC();
  for (int s = 0; s < steps; ++s) {
    bm_gemm(T1, k, Mj, k, false, P, k, false, k, k, k, 1.0, 0.0);      // T1 = Mj P
    bm_gemm(P, k, T1, k, false, Mj, k, true, k, k, k, 1.0, 1.0);       // P += T1 Mj'
    bm_gemm(T1, k, Mj, k, false, Mj, k, false, k, k, k, 1.0, 0.0);     // T1 = Mj Mj
    bm_copy(Mj, k, T1, k, k, k);
  }
  bm_symmetrize(P, k, k);
  for (int e = DFM_TID; e < kk; e += DFM_NT) P0all[(size_t)b * kk + e] = P[e];
}

// Per-iteration preparation: closes the previous iteration (convergence / iteration count) and builds
// W = Lam / R, logR, C = Lam' R^-1 Lam for the next E-step.  grid (B), one block.
__global__ void k_em_prep(const double* __restrict__ LamAll, const double* __restrict__ Rall, int N, int r, int p,
                          double* __restrict__ Wall, double* __restrict__ logRall, double* __restrict__ Call,
                          double* __restrict__ A, const double* __restrict__ Anew, double* __restrict__ Q,
                          const double* __restrict__ Qnew, EmState* st, int max_iter, int closing, int skip_bal) {
  int b = DFM_BX;
  if (closing && skip_bal && !st[b].has_missing) return;      // balanced panels are closed by k_emb_close
  int was_done = st[b].done;
  DFM_SYNC();
  if (closing && !was_done) {
    int rk = r * r * p, rr = r * r;                    // commit the transition M-step of this iteration
    for (int e = DFM_TID; e < rk; e += DFM_NT) A[(size_t)b * rk + e] = Anew[(size_t)b * rk + e];
    for (int e = DFM_TID; e < rr; e += DFM_NT) Q[(size_t)b * rr + e] = Qnew[(size_t)b * rr + e];
    if (DFM_TID == 0) {
      st[b].iters += 1;
      if (st[b].conv_pending || st[b].iters >= max_iter || st[b].status == 3) st[b].done = 1;
    }
    DFM_SYNC();
  }
  if (st[b].done) return;
  const double* Lam = LamAll + (size_t)b * N * r; const double* R = Rall + (size_t)b * N;
  double* W = Wall + (size_t)b * N * r; double* logR = logRall + (size_t)b * N; double* C = Call + (size_t)b * r * r;
  for (int i = DFM_TID; i < N; i += DFM_NT) {
    bool use = !is_nan(Lam[i]) && !is_nan(R[i]);
    double rinv = use ? 1.0 / R[i] : 0.0;
    for (int a = 0; a < r; ++a) W[i + (size_t)N * a] = use ? Lam[i + (size_t)N * a] * rinv : DFM_NAN;
    logR[i] = use ? log(R[i]) : 0.0;
    if (use && !(R[i] > 0.0)) st[b].status = 3;
  }
  DFM_SYNC();
  if (skip_bal && !st[b].has_missing) return;            // (initial call on the multi-CTA path: C comes from k_emb_cinit + k_emb_close)
  for (int e = DFM_TID; e < r * r; e += DFM_NT) {
    int a = e % r, c = e / r;
    if (a < c) continue;
    double s = 0.0;
    for (int i = 0; i < N; ++i) { double w = W[i + (size_t)N * a]; if (!is_nan(w)) s += w * Lam[i + (size_t)N * c]; }
    C[a + r * c] = s; C[c + r * a] = s;
  }
}

// E-step contraction: b_t = Lam' R^-1 x_t, q_t = x_t' R^-1 x_t, n_t, sum_obs log R_i and (when data are
// missing) the packed information matrix C_t = C - sum_{i missing} lam_i lam_i'/R_i.
// One THREAD per period t (coalesced column-major reads); per-thread workspace in shared memory.
// grid (ceil(T/NT), B); shared (r + np) * NT doubles.
__global__ void k_em_contract(const double* __restrict__ Xall, const double* __restrict__ LamAll,
                              const double* __restrict__ Wall, const double* __restrict__ Rall,
                              const double* __restrict__ logRall, const double* __restrict__ Call, int T, int N, int r,
                              double* __restrict__ Bt, double* __restrict__ qt, double* __restrict__ slr,
                              int* __restrict__ nt_, double* __restrict__ Ct, const EmState* st) {
  DFM_SMEM(sm);
  int b = DFM_BY;
  if (st[b].done || !st[b].has_missing) return;   // balanced panels: k_em_contract_bal
  int np = r * (r + 1) / 2, nt = DFM_NT;
  double* c = sm + DFM_TID;                       // c[a*nt]
  double* A = sm + (size_t)r * nt + DFM_TID;      // A[e*nt]
  const double* X = Xall + (size_t)b * T * N; const double* Lam = LamAll + (size_t)b * N * r;
  const double* W = Wall + (size_t)b * N * r; const double* R = Rall + (size_t)b * N;
  const double* logR = logRall + (size_t)b * N; const double* C = Call + (size_t)b * r * r;
  int hm = st[b].has_missing;
  for (int t = DFM_BX * nt + DFM_TID; t < T; t += DFM_GX * nt) {
    for (int a = 0; a < r; ++a) c[a * nt] = 0.0;
    if (hm) for (int a = 0; a < r; ++a) for (int cc = 0; cc <= a; ++cc) A[pidx(a, cc) * nt] = C[a + r * cc];
    double q = 0.0, sl = 0.0; int n = 0;
    for (int i = 0; i < N; ++i) {
      double w0 = W[i];
      if (is_nan(w0)) continue;                   // series excluded from the model
      double x = X[t + (size_t)T * i];
      if (!is_nan(x)) {
        ++n; q += x * x / R[i]; sl += logR[i];
        for (int a = 0; a < r; ++a) c[a * nt] += x * W[i + (size_t)N * a];
      } else if (hm) {
        for (int a = 0; a < r; ++a) { double wa = W[i + (size_t)N * a]; for (int cc = 0; cc <= a; ++cc) A[pidx(a, cc) * nt] -= wa * Lam[i + (size_t)N * cc]; }
      }
    }
    for (int a = 0; a < r; ++a) Bt[(size_t)b * T * r + t + (size_t)T * a] = c[a * nt];
    qt[(size_t)b * T + t] = q; slr[(size_t)b * T + t] = sl; nt_[(size_t)b * T + t] = n;
    if (hm) for (int e = 0; e < np; ++e) Ct[(size_t)b * T * np + t + (size_t)T * e] = A[e * nt];
  }
}

// max over the block of two values at once.  red: >= 80 doubles of shared scratch.  All threads get the results.
__device__ __forceinline__ void block_max2(double& a, double& b, double* red) {
#ifndef DFM_EMU
  for (int o = 16; o > 0; o >>= 1) { a = fmax(a, __shfl_xor_sync(0xffffffffu, a, o)); b = fmax(b, __shfl_xor_sync(0xffffffffu, b, o)); }
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  if (lane == 0) { red[w] = a; red[40 + w] = b; }
  __syncthreads();
  double x = red[0], y = red[40];
  for (int i = 1; i < nw; ++i) { x = fmax(x, red[i]); y = fmax(y, red[40 + i]); }
  __syncthreads();
  a = x; b = y;
#else
  (void)red;
#endif
}

// E-step contraction of a BALANCED panel (no NaN among the series in the model): b_t = W' x_t, q_t, sum log R, n_t; the
// information matrix is the constant C.  32 periods x 8 component groups per block: lane = period (coalesced reads of
// the column-major panel), warp = component group g (components g, g + 8, ...: the W loads are warp-uniform broadcasts).
// r <= 64.  grid (ceil(T / 32), B), 256 threads.
__global__ void k_em_contract_bal(const double* __restrict__ Xall, const double* __restrict__ Wall, const double* __restrict__ Rall,
                                  const double* __restrict__ logRall, int T, int N, int r, double* __restrict__ Bt,
                                  double* __restrict__ qt, double* __restrict__ slr, int* __restrict__ nt_, const EmState* st) {
  DFM_SMEM(part);                                 // [8][32][3] partial (q, sum log R, n) of the component groups
  int b = DFM_BY;
  if (st[b].done || st[b].has_missing) return;
  const double* X = Xall + (size_t)b * T * N; const double* W = Wall + (size_t)b * N * r;
  const double* R = Rall + (size_t)b * N; const double* logR = logRall + (size_t)b * N;
  for (int idx = DFM_TID; idx < 256; idx += DFM_NT) {
    const int tl = idx & 31, g = idx >> 5, t = DFM_BX * 32 + tl;
    double acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.0;
    double q = 0.0, sl = 0.0, n = 0.0;
    if (t < T)
      for (int i = 0; i < N; ++i) {
        if (is_nan(W[i])) continue;               // series excluded from the model (uniform over the block)
        const double x = X[t + (size_t)T * i];
#pragma unroll
        for (int j = 0; j < 8; ++j) { const int a = g + 8 * j; if (a < r) acc[j] += x * W[i + (size_t)N * a]; }
        if ((i & 7) == g) { n += 1.0; q += x * x / R[i]; sl += logR[i]; }       // the scalar sums are split over the groups
      }
    if (t < T) {
#pragma unroll
      for (int j = 0; j < 8; ++j) { const int a = g + 8 * j; if (a < r) Bt[(size_t)b * T * r + t + (size_t)T * a] = acc[j]; }
    }
    part[(g * 32 + tl) * 3] = q; part[(g * 32 + tl) * 3 + 1] = sl; part[(g * 32 + tl) * 3 + 2] = n;
  }
  DFM_SYNC();
  for (int tl = DFM_TID; tl < 32; tl += DFM_NT) {
    const int t = DFM_BX * 32 + tl;
    if (t >= T) continue;
    double q = 0.0, sl = 0.0, n = 0.0;
    for (int g = 0; g < 8; ++g) { q += part[(g * 32 + tl) * 3]; sl += part[(g * 32 + tl) * 3 + 1]; n += part[(g * 32 + tl) * 3 + 2]; }
    qt[(size_t)b * T + t] = q; slr[(size_t)b * T + t] = sl; nt_[(size_t)b * T + t] = (int)n;
  }
}

// ---- small dense helpers of the filter / smoother steps ------------------------------------------------------------
// ---- parallel-in-time treatment of FROZEN RUNS (consecutive periods whose covariances are the stored steady state):
// the mean recursion  z_t = Phi z_{t -+ 1} + u_t  with a constant k x k matrix is a linear scan.  The run is cut into
// EM_RUN_NCH chunks, one per warp: pass 1 = chunk-local recursion from a zero state (keeps only the end state),
// boundary propagation with Phi^Lc (binary powering, block-cooperative), pass 2 = the recursion again from the true
// incoming state, writing z_t over u_t in place.  The u_t of the next four steps are prefetched into registers (they
// come from L2; the recursion itself runs out of shared memory).  C3 (T = 2000, k = 20): 2 x 2000 serial steps -> 2 x 2 x 125.
#define EM_RUN_NCH 16          // chunks per run (= warps used by the scan)
#define EM_RUN_MIN 32          // shorter runs take the serial frozen steps

// zg: global [T][k] (u_t in, z_t out) ; the run covers L periods starting at t_first and moving in direction dir (+1 / -1);
// Phi: k x k column-major (shared) ; z_in: state entering the run (k) ; Rp, base, tmp: k x k shared temporaries ;
// wb: 3 * k * EM_RUN_NCH doubles of shared workspace.  k <= 64.  Ends with a block barrier.
#ifdef DFM_EMU
#define EM_NOINLINE
#else
#define EM_NOINLINE __noinline__
#endif
// ---- thread-block CLUSTER per panel (few panels, e.g. C3): the CTAs of a cluster run the serial parts (explicit steps,
// boundary chain) redundantly -- same inputs, same arithmetic, same results -- and split the parallel parts of the frozen
// runs (tiles of the element-wise phases, chunks of the scan) by cluster rank; they exchange through global memory +
// cluster barriers (barrier.cluster arrive.release / wait.acquire after a fence).  A plain launch is a cluster of one.
#ifndef DFM_EMU
__device__ __forceinline__ int cl_rank() { unsigned r_; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r_)); return (int)r_; }
__device__ __forceinline__ int cl_size() { unsigned r_; asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(r_)); return (int)r_; }
__device__ __forceinline__ void cl_sync(int nc) {
  if (nc > 1) {
    __threadfence();
    asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
    asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
  }
}
#else
__device__ __forceinline__ int cl_rank() { return 0; }
__device__ __forceinline__ int cl_size() { return 1; }
__device__ __forceinline__ void cl_sync(int) {}
#endif

#ifndef DFM_EMU
// Tensor-core variant of the run scan for k <= 32 and a large workspace (one CTA per SM configurations): 64 chunks, 8 per warp
// on warps 0..7.  A warp advances its 8 chunk recursions together: the step  Z <- Phi Z + U  with Z = [k x 8 chunks] is
// ceil(k/8) x ceil(k/4) DMMA.8x8x4 with the Phi fragments in registers and Z as the B operand from a [k][12] shared tile
// (conflict-free); the u_t of later steps are pulled into L1 four steps ahead (prefetch.global.L1).  A step costs one
// dependent DMMA chain (~ceil(k/4) DMMA latencies) instead of ~100 instructions per chunk, and the chains are 4x shorter
// (64 chunks).  ws: >= 256 k doubles of shared workspace.
#define EM_SC_NW 8
#define EM_SC_ZS 12
template <int MB>
__device__ EM_NOINLINE void em_run_scan_tc(double* __restrict__ zg, int k, int t_first, int L, int dir, const double* Phi,
                                           const double* z_in, double* Rp, double* base, double* tmp, double* ws, int nc, int crank,
                                           double* xbnd) {
  constexpr int KBX = 2 * MB, KR = 8 * MB;             // k-chunks and (zero padded) state rows of a warp's tile
  const int NCH = 8 * EM_SC_NW;
  const int Lc = (L + NCH - 1) / NCH;
  // Rp = Phi^Lc (binary powering on the tensor path; the three buffers rotate)
  for (int e = DFM_TID; e < k * k; e += DFM_NT) { int i = e % k, j = e / k; Rp[e] = (i == j) ? 1.0 : 0.0; base[e] = Phi[e]; }
  DFM_SYNC();
  for (int ex = Lc; ex > 0; ex >>= 1) {
    if (ex & 1) {
      wt_gemm(Rp, 1, k, base, k, 1, k, k, k, [&](int i, int j, double v) { tmp[i + k * j] = v; });
      DFM_SYNC();
      double* sw = Rp; Rp = tmp; tmp = sw;
    }
    if (ex > 1) {
      wt_gemm(base, 1, k, base, k, 1, k, k, k, [&](int i, int j, double v) { tmp[i + k * j] = v; });
      DFM_SYNC();
      double* sw = base; base = tmp; tmp = sw;
    }
  }
  double* bnd = ws + (size_t)EM_SC_NW * 2 * KR * EM_SC_ZS;             // [64][k]: e_c, then in_c
  const int lr = DFM_LANE >> 2, lc = DFM_LANE & 3, wl = DFM_WARP;
  const int w = wl * nc + crank;                        // virtual warp of the cluster: 8 chunks each, EM_SC_NW in total
  for (int pass = 1; pass <= 2; ++pass) {
    if (w < EM_SC_NW) {
      double* cur = ws + (size_t)wl * 2 * KR * EM_SC_ZS; double* nxt = cur + (size_t)KR * EM_SC_ZS;
      double aP[MB][KBX];
#pragma unroll
      for (int mb = 0; mb < MB; ++mb)
#pragma unroll
        for (int kb = 0; kb < KBX; ++kb) {
          const int i = mb * 8 + lr, l = kb * 4 + lc;
          aP[mb][kb] = (i < k && l < k) ? Phi[i + k * l] : 0.0;
        }
      // this lane's two chunks (columns 2 lc, 2 lc + 1 of the warp's tile) and their first periods
      const int cA = 8 * w + 2 * lc, cB = cA + 1;
      const long long tA = (long long)t_first + (long long)dir * cA * Lc, tB = (long long)t_first + (long long)dir * cB * Lc;
      const int lenA = (L - cA * Lc < Lc) ? ((L - cA * Lc > 0) ? L - cA * Lc : 0) : Lc;
      const int lenB = (L - cB * Lc < Lc) ? ((L - cB * Lc > 0) ? L - cB * Lc : 0) : Lc;
      const long long dk = (long long)dir * k;
      bool rok[MB];
#pragma unroll
      for (int mb = 0; mb < MB; ++mb) rok[mb] = mb * 8 + lr < k;
      for (int e = DFM_LANE; e < KR * 8; e += 32) {     // (rows >= k stay zero in both buffers: no bounds tests in the step)
        const int i = e >> 3, n = e & 7;
        cur[i * EM_SC_ZS + n] = (pass == 1 || i >= k) ? 0.0 : bnd[(size_t)(8 * w + n) * k + i];
        nxt[i * EM_SC_ZS + n] = 0.0;
      }
      __syncwarp();
      double* pA = zg + tA * k + lr; double* pB = zg + tB * k + lr;
      // u_t of two steps ahead in registers (an L2 round trip is longer than a step; prefetch.global.L1 did not hide it)
      double cuA[2][MB], cuB[2][MB];
#pragma unroll
      for (int q = 0; q < 2; ++q)
#pragma unroll
        for (int mb = 0; mb < MB; ++mb) {
          cuA[q][mb] = (rok[mb] && q < lenA) ? pA[q * dk + mb * 8] : 0.0;
          cuB[q][mb] = (rok[mb] && q < lenB) ? pB[q * dk + mb * 8] : 0.0;
        }
      for (int s2 = 0; s2 < Lc; s2 += 2) {
        double nA[2][MB], nB[2][MB];
#pragma unroll
        for (int q = 0; q < 2; ++q)
#pragma unroll
          for (int mb = 0; mb < MB; ++mb) {
            const int sn = s2 + 2 + q;
            nA[q][mb] = (rok[mb] && sn < lenA) ? pA[sn * dk + mb * 8] : 0.0;
            nB[q][mb] = (rok[mb] && sn < lenB) ? pB[sn * dk + mb * 8] : 0.0;
          }
#pragma unroll
        for (int q = 0; q < 2; ++q) {
          const int s_ = s2 + q;
          if (s_ < Lc) {
            const bool okA = s_ < lenA, okB = s_ < lenB;
            double* gA = pA + s_ * dk; double* gB = pB + s_ * dk;
            double d[MB][2];
#pragma unroll
            for (int mb = 0; mb < MB; ++mb) { d[mb][0] = 0.0; d[mb][1] = 0.0; }
            double bz[KBX];
#pragma unroll
            for (int kb = 0; kb < KBX; ++kb) bz[kb] = cur[(kb * 4 + lc) * EM_SC_ZS + lr];
#pragma unroll
            for (int kb = 0; kb < KBX; ++kb)
#pragma unroll
              for (int mb = 0; mb < MB; ++mb) EM_DMMA(d[mb], aP[mb][kb], bz[kb]);
#pragma unroll
            for (int mb = 0; mb < MB; ++mb) {
              const int i = mb * 8 + lr;
              const double vA = d[mb][0] + cuA[q][mb], vB = d[mb][1] + cuB[q][mb];
              nxt[i * EM_SC_ZS + 2 * lc] = vA; nxt[i * EM_SC_ZS + 2 * lc + 1] = vB;       // (rows >= k: 0 + 0)
              if (pass == 2 && rok[mb]) {
                if (okA) gA[mb * 8] = vA;
                if (okB) gB[mb * 8] = vB;
              }
            }
            __syncwarp();
            double* sw = cur; cur = nxt; nxt = sw;
          }
        }
#pragma unroll
        for (int q = 0; q < 2; ++q)
#pragma unroll
          for (int mb = 0; mb < MB; ++mb) { cuA[q][mb] = nA[q][mb]; cuB[q][mb] = nB[q][mb]; }
      }
      if (pass == 1) {
        double* dst = (nc > 1) ? xbnd : bnd;             // (cluster: end states go through global memory)
        for (int e = DFM_LANE; e < k * 8; e += 32) { const int i = e >> 3, n = e & 7; dst[(size_t)(8 * w + n) * k + i] = cur[i * EM_SC_ZS + n]; }
      }
    }
    DFM_SYNC();
    cl_sync(nc);
    if (pass == 1) {
      if (nc > 1) { for (int e = DFM_TID; e < NCH * k; e += DFM_NT) bnd[e] = xbnd[e]; DFM_SYNC(); }
      // incoming states on warp 0: in_0 = z_in, in_{c+1} = Phi^Lc in_c + e_c  (row i of Phi^Lc in the registers of lane i,
      // zero padded to 32 x 32 so that the step has no bounds tests; bnd[c] is overwritten by in_c)
      if (wl == 0) {
        double* inc = ws;                               // 32 doubles (warp 0's idle tile)
        const int i = DFM_LANE;
        const bool iok = i < k;
        double rw[32];
#pragma unroll
        for (int j = 0; j < 32; ++j) rw[j] = (iok && j < k) ? Rp[i + k * j] : 0.0;
        inc[i] = iok ? z_in[i] : 0.0;
        __syncwarp();
        for (int c = 0; c < NCH; ++c) {
          double a0 = 0.0, a1 = 0.0, a2 = 0.0, a3 = 0.0;
#pragma unroll
          for (int j = 0; j < 32; j += 4) { a0 += rw[j] * inc[j]; a1 += rw[j + 1] * inc[j + 1]; a2 += rw[j + 2] * inc[j + 2]; a3 += rw[j + 3] * inc[j + 3]; }
          const double ec = iok ? bnd[(size_t)c * k + i] : 0.0, ic = inc[i];
          __syncwarp();
          if (iok) bnd[(size_t)c * k + i] = ic;
          inc[i] = ((a0 + a1) + (a2 + a3)) + ec;        // (lanes >= k: 0)
          __syncwarp();
        }
      }
      DFM_SYNC();
    }
  }
}
#endif

__device__ EM_NOINLINE void em_run_scan(double* __restrict__ zg, int k, int t_first, int L, int dir, const double* Phi,
                                   const double* z_in, double* Rp, double* base, double* tmp, double* wb, double* ws, int ws_doubles,
                                   int nc, int crank, double* xbnd) {
#ifndef DFM_EMU
  if (k <= 32 && DFM_NWARP >= EM_SC_NW && ws_doubles >= EM_SC_NW * 2 * 8 * ((k + 7) >> 3) * EM_SC_ZS + 8 * EM_SC_NW * k && L >= 256) {
    switch ((k + 7) >> 3) {
      case 1: em_run_scan_tc<1>(zg, k, t_first, L, dir, Phi, z_in, Rp, base, tmp, ws, nc, crank, xbnd); break;
      case 2: em_run_scan_tc<2>(zg, k, t_first, L, dir, Phi, z_in, Rp, base, tmp, ws, nc, crank, xbnd); break;
      case 3: em_run_scan_tc<3>(zg, k, t_first, L, dir, Phi, z_in, Rp, base, tmp, ws, nc, crank, xbnd); break;
      default: em_run_scan_tc<4>(zg, k, t_first, L, dir, Phi, z_in, Rp, base, tmp, ws, nc, crank, xbnd); break;
    }
    return;
  }
#else
  (void)ws; (void)ws_doubles;
#endif
  (void)nc; (void)crank; (void)xbnd;                   // (this variant is not split: the CTAs of a cluster run it redundantly)
  const int Lc = (L + EM_RUN_NCH - 1) / EM_RUN_NCH;
  // Rp = Phi^Lc
  for (int e = DFM_TID; e < k * k; e += DFM_NT) { int i = e % k, j = e / k; Rp[e] = (i == j) ? 1.0 : 0.0; base[e] = Phi[e]; }
  DFM_SYNC();
  for (int ex = Lc; ex > 0; ex >>= 1) {
    if (ex & 1) { bm_gemm(tmp, k, Rp, k, false, base, k, false, k, k, k, 1.0, 0.0); bm_copy(Rp, k, tmp, k, k, k); }
    if (ex > 1) { bm_gemm(tmp, k, base, k, false, base, k, false, k, k, k, 1.0, 0.0); bm_copy(base, k, tmp, k, k, k); }
  }
  for (int pass = 1; pass <= 2; ++pass) {
    for (int c = DFM_WARP; c < EM_RUN_NCH; c += DFM_NWARP) {
      double* cur = wb + (size_t)c * 3 * k; double* nxt = cur + k; double* bnd = cur + 2 * k;
      const int s0 = c * Lc, len = (L - s0 < Lc) ? ((L - s0 > 0) ? L - s0 : 0) : Lc;
      for (int i = DFM_LANE; i < k; i += DFM_WSZ) cur[i] = (pass == 1) ? 0.0 : bnd[i];
      DFM_WSYNC();
      // rows of this lane: i0 = lane, i1 = lane + warp size (k <= 2 warp sizes on the GPU; the emulation loops over rows)
#ifndef DFM_EMU
      const int i0 = DFM_LANE, i1 = DFM_LANE + 32;
      const bool r0 = i0 < k, r1 = i1 < k;
      if (k <= 32) {
        // row i0 of Phi in registers: a step costs k broadcast reads of the state instead of 2 k^2 / 32 operand reads per lane
        // (16 warps running this from shared-memory operands alone saturate the shared-memory pipe)
        double ph[32];
#pragma unroll
        for (int j = 0; j < 32; ++j) ph[j] = (r0 && j < k) ? Phi[i0 + k * j] : 0.0;
        double ub[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) { const long long tt = t_first + (long long)dir * (s0 + q); ub[q] = (q < len && r0) ? zg[tt * k + i0] : 0.0; }
        for (int sg = 0; sg < len; sg += 4) {
          double un[4];
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const int sn = sg + 4 + q;
            const long long tt = t_first + (long long)dir * (s0 + sn);
            un[q] = (sn < len && r0) ? zg[tt * k + i0] : 0.0;
          }
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            if (sg + q < len) {
              const long long tt = t_first + (long long)dir * (s0 + sg + q);
              double a0 = 0.0, a1 = 0.0, a2 = 0.0, a3 = 0.0;
#pragma unroll
              for (int j = 0; j < 32; j += 4) {
                if (j < k) {
                  a0 += ph[j] * cur[j];
                  if (j + 1 < k) a1 += ph[j + 1] * cur[j + 1];
                  if (j + 2 < k) a2 += ph[j + 2] * cur[j + 2];
                  if (j + 3 < k) a3 += ph[j + 3] * cur[j + 3];
                }
              }
              if (r0) { const double v = ((a0 + a1) + (a2 + a3)) + ub[q]; nxt[i0] = v; if (pass == 2) zg[tt * k + i0] = v; }
              __syncwarp();
              double* sw = cur; cur = nxt; nxt = sw;
            }
          }
#pragma unroll
          for (int q = 0; q < 4; ++q) ub[q] = un[q];
        }
      } else {
      double ub0[4], ub1[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const long long tt = t_first + (long long)dir * (s0 + q);
        ub0[q] = (q < len && r0) ? zg[tt * k + i0] : 0.0; ub1[q] = (q < len && r1) ? zg[tt * k + i1] : 0.0;
      }
      for (int sg = 0; sg < len; sg += 4) {
        double un0[4], un1[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int sn = sg + 4 + q;
          const long long tt = t_first + (long long)dir * (s0 + sn);
          un0[q] = (sn < len && r0) ? zg[tt * k + i0] : 0.0; un1[q] = (sn < len && r1) ? zg[tt * k + i1] : 0.0;
        }
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          if (sg + q < len) {
            const long long tt = t_first + (long long)dir * (s0 + sg + q);
            double a0 = 0.0, a1 = 0.0, c0 = 0.0, c1 = 0.0;
            int j = 0;
            for (; j + 1 < k; j += 2) {
              const double z0 = cur[j], z1 = cur[j + 1];
              if (r0) { a0 += Phi[i0 + k * j] * z0; a1 += Phi[i0 + k * (j + 1)] * z1; }
              if (r1) { c0 += Phi[i1 + k * j] * z0; c1 += Phi[i1 + k * (j + 1)] * z1; }
            }
            if (j < k) { const double z0 = cur[j]; if (r0) a0 += Phi[i0 + k * j] * z0; if (r1) c0 += Phi[i1 + k * j] * z0; }
            if (r0) { const double v = (a0 + a1) + ub0[q]; nxt[i0] = v; if (pass == 2) zg[tt * k + i0] = v; }
            if (r1) { const double v = (c0 + c1) + ub1[q]; nxt[i1] = v; if (pass == 2) zg[tt * k + i1] = v; }
            __syncwarp();
            double* sw = cur; cur = nxt; nxt = sw;
          }
        }
#pragma unroll
        for (int q = 0; q < 4; ++q) { ub0[q] = un0[q]; ub1[q] = un1[q]; }
      }
      }
#else
      for (int s_ = 0; s_ < len; ++s_) {
        const int tt = t_first + dir * (s0 + s_);
        for (int i = 0; i < k; ++i) {
          double a0 = 0.0;
          for (int j = 0; j < k; ++j) a0 += Phi[i + k * j] * cur[j];
          const double v = a0 + zg[(size_t)tt * k + i];
          nxt[i] = v;
          if (pass == 2) zg[(size_t)tt * k + i] = v;
        }
        double* sw = cur; cur = nxt; nxt = sw;
      }
#endif
      if (pass == 1) {                                  // end state of the zero-start recursion -> bnd (cur may be either buffer)
        double* b0 = wb + (size_t)c * 3 * k + 2 * k;
        for (int i = DFM_LANE; i < k; i += DFM_WSZ) b0[i] = cur[i];
      }
    }
    DFM_SYNC();
    if (pass == 1) {
      // incoming states: in_0 = z_in, in_{c+1} = Phi^Lc in_c + e_c ; bnd[c] holds e_c and is overwritten by in_c
      double* inc = wb;                                  // 2k doubles (chunk 0's idle cur/nxt buffers): current in_c, next in_c
      for (int i = DFM_TID; i < k; i += DFM_NT) inc[i] = z_in[i];
      DFM_SYNC();
      for (int c = 0; c + 1 < EM_RUN_NCH; ++c) {
        double* ec = wb + (size_t)c * 3 * k + 2 * k;
        for (int i = DFM_TID; i < k; i += DFM_NT) { double s = ec[i]; for (int j = 0; j < k; ++j) s += Rp[i + k * j] * inc[j]; inc[k + i] = s; }
        DFM_SYNC();
        for (int i = DFM_TID; i < k; i += DFM_NT) { ec[i] = inc[i]; inc[i] = inc[k + i]; }      // bnd[c] <- in_c
        DFM_SYNC();
      }
      double* el = wb + (size_t)(EM_RUN_NCH - 1) * 3 * k + 2 * k;
      for (int i = DFM_TID; i < k; i += DFM_NT) el[i] = inc[i];
      DFM_SYNC();
    }
  }
}

// shared-memory footprint (doubles) of k_em_filter_smooth; stg_T = periods per staging tile of the frozen-run phases
__host__ __device__ inline size_t em_fs_smem_doubles(int r, int p, int stg_T = 16) {
  size_t k = (size_t)r * p, kk = k * k, rr = (size_t)r * r, rk = (size_t)r * k;
  return 9 * kk + 7 * rr + 3 * rk + 6 * k + 2 * r + 64 + 64 + 3 * k * EM_RUN_NCH + (size_t)r * (stg_T + 4) + (size_t)(2 * stg_T + 1) * em_lds((int)k) + 8 + 3 * 64;
}

#ifdef DFM_EMU
#define EM_FS_BOUNDS
#else
#define EM_FS_BOUNDS __launch_bounds__(512, 1)
#endif
#define EM_ACC_MAX 8           // Gram-sum outputs per thread held in registers by the backward frozen runs

// Kalman filter + RTS smoother + transition M-step for one panel.  grid (B), one block (256 or 512 threads).
// Scratch (global, per panel): zp, zf [T x k]; Pp, Pf [T x k x k].
// Outputs: Fs [T x r], PsF packed [T x np] (smoothed Var f_t), SffAll [r x r] = sum_t E f f',
// Anew [r x k], Qnew [r x r], loglik path.
//
// EXPLICIT STEPS (covariances move).  Forward, information form: P_{t|t-1} from the companion structure of M (rows >= r
// of M are a shift: only A P_f, r k^2 flops, is a product), Cholesky factors of P_ff and S = I + L'C L on warp 0 with
// warp barriers, the two triangular solves on transposed right-hand sides (thread per row, no barriers, conflict-free).
// Backward: J = P_f M' P_p^-1 is obtained row-wise the same way (right-hand sides = rows of P_f M'), so only J -- never
// J' -- is needed: zs = zf + J dv, Ps = Pf + (J D) J', Pc = Ps(t+1)[0:r,:] J' are all conflict-free products.
// FROZEN STEPS.  Where the information matrix C_t does not change (a balanced panel: everywhere; missing data: between
// two changes of the observation pattern) the covariance recursion is data independent and converges to its steady
// state; once P_{t|t-1} repeats (relative 1e-14) the factorisations, the gain and P_{t|t} of the following periods
// are the ones already in shared memory, and only the mean updates remain: serial steps for short runs, the parallel
// scan above for runs of >= EM_RUN_MIN periods (inputs and outputs of the element-wise phases staged through shared
// memory in tiles of stg_T periods).  src[t] = the period whose stored covariances period t uses.  The smoother gain
// and the smoothed covariance freeze the same way.
__global__ void EM_FS_BOUNDS k_em_filter_smooth(const double* __restrict__ Aall, const double* __restrict__ Qall,
                                   const double* __restrict__ P0all, const double* __restrict__ Call,
                                   const double* __restrict__ Bt_, const double* __restrict__ qt_,
                                   const double* __restrict__ slr_, const int* __restrict__ nt__,
                                   const double* __restrict__ Ct_, int T, int r, int p,
                                   double* __restrict__ zp_, double* __restrict__ zf_, double* __restrict__ Pp_,
                                   double* __restrict__ Pf_, double* __restrict__ Fs_, double* __restrict__ PsF_,
                                   double* __restrict__ SffAll_, double* __restrict__ Anew_, double* __restrict__ Qnew_,
                                   double* __restrict__ loglik_, int max_iter, double tol, EmState* st, int* __restrict__ src_,
                                   int stg_T, int want_psf, double* __restrict__ xch_) {
  DFM_SMEM(sm);
  const int NC = cl_size(), crank = cl_rank();           // cluster per panel (1 for a plain launch)
  int b = DFM_BX / NC;
  if (st[b].done) return;
  int k = r * p, kk = k * k, rr = r * r, rk = r * k, np = r * (r + 1) / 2;
  double* M = sm;            double* Pp = M + kk;      double* Pf = Pp + kk;    double* T1 = Pf + kk;
  double* T2 = T1 + kk;      double* T3 = T2 + kk;     double* Psn = T3 + kk;   double* S00 = Psn + kk;
  double* Ps = S00 + kk;
  double* Q = Ps + kk;       double* C = Q + rr;       double* L = C + rr;      double* S = L + rr;
  double* Sff2 = S + rr;     double* SffA = Sff2 + rr; double* T4 = SffA + rr;
  double* Tm = T4 + rr;      double* Wm = Tm + rk;     double* S11 = Wm + rk;
  double* zp = S11 + rk;     double* zf = zp + k;      double* zsn = zf + k;    double* zs = zsn + k;
  double* dv = zs + k;       double* tv = dv + k;
  double* g = tv + k;        double* bt = g + r;
  double* red = bt + r;      // 40 (+ 80 for block_max2 behind `info`)
  int* info = (int*)(red + 44);                          // [0] Cholesky flag, [1] run search, [2], [3]: "C changed" flags of even / odd periods
  double* red2 = red + 48;   // 80
  double* wb = red2 + 80;    // 3 * k * EM_RUN_NCH: scan workspace of the frozen runs
  double* stg = wb + 3 * k * EM_RUN_NCH;   // stg_T * (2k + r) + 2k: staging tiles of the frozen-run phases
  const int stg_doubles = r * (stg_T + 4) + (2 * stg_T + 1) * em_lds(k) + 8;
  double* dvL = stg + stg_doubles;   // 1 / diag of the Cholesky factors: L (or Pp), S
  double* dvS = dvL + 64;
  double* ldS_sh = red + 40; // log det of the last explicit step, for all threads
  int* src = src_ + (size_t)b * T;
  // cluster exchange buffers of this panel (global): [0..15] scalars by rank, then 64 k boundary states, then NC x (kk + rk) Gram partials
  double* xch = xch_ ? xch_ + (size_t)b * (16 + 64 * (size_t)k + 16 * ((size_t)kk + rk)) : nullptr;
  double* xbnd = xch ? xch + 16 : nullptr;
  double* xgram = xch ? xch + 16 + 64 * (size_t)k : nullptr;
  const double* A = Aall + (size_t)b * rk; const double* Qg = Qall + (size_t)b * rr;
  const double* P0 = P0all + (size_t)b * kk; const double* Cg = Call + (size_t)b * rr;
  const double* Bt = Bt_ + (size_t)b * T * r; const double* qt = qt_ + (size_t)b * T;
  const double* slr = slr_ + (size_t)b * T; const int* ntv = nt__ + (size_t)b * T;
  const double* Ct = Ct_ + (size_t)b * T * np;
  double* zpg = zp_ + (size_t)b * T * k; double* zfg = zf_ + (size_t)b * T * k;
  double* Ppg = Pp_ + (size_t)b * T * kk; double* Pfg = Pf_ + (size_t)b * T * kk;
  double* Fs = Fs_ + (size_t)b * T * r; double* PsF = PsF_ + (size_t)b * T * np;
  int hm = st[b].has_missing;
  const int TT = stg_T;
  const bool psf = hm || want_psf;       // the smoothed covariances leave the kernel only if the M-step (missing data) or the caller needs them
  if (DFM_TID == 0) { info[0] = 0; info[1] = 0; info[2] = 0; info[3] = 0; }
  for (int e = DFM_TID; e < kk; e += DFM_NT) {
    int i = e % k, j = e / k;
    M[e] = (i < r) ? A[i + r * j] : ((j == i - r) ? 1.0 : 0.0);
    S00[e] = 0.0;
  }
  for (int e = DFM_TID; e < rr; e += DFM_NT) { Q[e] = Qg[e]; C[e] = Cg[e]; Sff2[e] = 0.0; SffA[e] = 0.0; }
  for (int e = DFM_TID; e < rk; e += DFM_NT) S11[e] = 0.0;
  DFM_SYNC();
  double ll = 0.0;
  // ------------------------------------------------------------------ forward: Kalman filter
  int frozen = 0, last_src = 0, run_known = 0;   // (uniform over the block; run_known: the frozen run in progress ends there)
  double ldS = 0.0;                      // thread 0: 2 sum log diag chol(S) of the last explicit step
  for (int t = 0; t < T; ++t) {
    // information matrix of this period; did it change?  (flag of this period's parity; thread 0 clears the other one)
    if (DFM_TID == 0) info[2 + ((t + 1) & 1)] = 0;
    if (hm) {
      for (int e = DFM_TID; e < rr; e += DFM_NT) {
        int a = e % r, c = e / r;
        double cn = (a >= c) ? Ct[t + (size_t)T * pidx(a, c)] : Ct[t + (size_t)T * pidx(c, a)];
        if (cn != C[e]) info[2 + (t & 1)] = 1;
        C[e] = cn;
      }
    }
    for (int e = DFM_TID; e < r; e += DFM_NT) bt[e] = Bt[t + (size_t)T * e];
    DFM_SYNC();
    const int cchg = (t == 0) ? 1 : info[2 + (t & 1)];
    if (frozen && !cchg && t >= run_known) {
      // ---- how far does this frozen run reach?  (next change of the information matrix, or T)
      int t1 = T;
      if (hm) {
        if (DFM_TID == 0) info[1] = T;
        DFM_SYNC();
        for (int base_ = t + 1; base_ < T; base_ += DFM_NT) {
          const int tp = base_ + DFM_TID;
          if (tp < T) {
            bool ch = false;
            for (int e = 0; e < np; ++e) ch = ch || (Ct[tp + (size_t)T * e] != Ct[tp - 1 + (size_t)T * e]);
            if (ch) atomicMin(&info[1], tp);
          }
          DFM_SYNC();
          const int v = info[1];
          DFM_SYNC();
          if (v < T) break;
        }
        t1 = info[1];
      }
      run_known = t1;
      const int Lr = t1 - t;
      if (Lr >= EM_RUN_MIN) {
        // ---- parallel frozen run [t, t1):  zf_t = Phi zf_{t-1} + Kb b_t,  Phi = M - Kb C M[0:r,:],  Kb = Pf[:, 0:r]
        bm_gemm(Tm, r, C, r, false, M, k, false, r, k, r, 1.0, 0.0);             // C M[0:r,:]   (Tm, Wm: rebuilt by the next explicit step)
        bm_gemm(T1, k, Pf, k, false, Tm, r, false, k, k, r, 1.0, 0.0);           // Kb (C M[0:r,:])
        for (int e = DFM_TID; e < kk; e += DFM_NT) T1[e] = M[e] - T1[e];
        const int TTp = TT + 4, lds = em_lds(k);
        double* Bs = stg;                           // [r][TTp]        b_t of the tile (component-major)
        double* Zs = Bs + (size_t)r * TTp;          // [TT + 1][lds]   zf_{t0-1} .. zf_{t0+len-1}
        double* Zq = Zs + (size_t)(TT + 1) * lds;   // [TT][lds]       zp of the tile
        for (int t0 = t, ti = 0; t0 < t1; t0 += TT, ++ti) {                      // u_t = Kb b_t  -> zfg
          if (ti % NC != crank) continue;                                        // (tiles dealt to the CTAs of the cluster)
          const int len = (t1 - t0 < TT) ? t1 - t0 : TT;
          DFM_SYNC();
#pragma unroll 4
          for (int e = DFM_TID; e < r * len; e += DFM_NT) { const int a = e / len, tt = e - a * len; Bs[a * TTp + tt] = Bt[t0 + tt + (size_t)T * a]; }
          DFM_SYNC();
          wt_gemm(Bs, 1, TTp, Pf, 1, k, len, k, r, [&](int m, int n, double v) { zfg[(size_t)(t0 + m) * k + n] = v; });
        }
        DFM_SYNC();
        cl_sync(NC);
        em_run_scan(zfg, k, t, Lr, +1, T1, zf, T2, T3, Psn, wb, stg, stg_doubles, NC, crank, xbnd);   // (T2, T3, Psn are free between explicit steps)
        cl_sync(NC);
        double llp = 0.0;
        const double ldS_ = *ldS_sh;
        for (int t0 = t, ti = 0; t0 < t1; t0 += TT, ++ti) {                      // zp_t = M zf_{t-1}, likelihood terms
          if (ti % NC != crank) continue;
          const int len = (t1 - t0 < TT) ? t1 - t0 : TT;
          DFM_SYNC();
#pragma unroll 4
          for (int e = DFM_TID; e < r * len; e += DFM_NT) { const int a = e / len, tt = e - a * len; Bs[a * TTp + tt] = Bt[t0 + tt + (size_t)T * a]; }
          {
            const double* g0 = zfg + (size_t)(t0 - 1) * k;                      // rows t0-1 .. t0+len-1 are contiguous
#pragma unroll 4
            for (int e = DFM_TID; e < (len + 1) * k; e += DFM_NT) {
              const int tt = e / k, i = e - tt * k;
              Zs[tt * lds + i] = (t0 == t && tt == 0) ? zf[i] : g0[e];
            }
          }
          DFM_SYNC();
          wt_gemm(Zs, lds, 1, M, 1, k, len, k, k, [&](int m, int n, double v) { Zq[m * lds + n] = v; zpg[(size_t)(t0 + m) * k + n] = v; });
          DFM_SYNC();
          wt_gemm(Zq, lds, 1, C, 1, r, len, r, r, [&](int m, int a, double cz) {
            const double ba = Bs[a * TTp + m], ga = ba - cz, zpa = Zq[m * lds + a], zfa = Zs[(m + 1) * lds + a];
            double term = -2.0 * zpa * ba + zpa * (ba - ga) - ga * (zfa - zpa);
            if (a == 0) { term += (double)ntv[t0 + m] * DFM_LOG2PI + slr[t0 + m] + ldS_ + qt[t0 + m]; src[t0 + m] = last_src; }
            llp += -0.5 * term;
          });
        }
        if (NC > 1) {                                      // likelihood terms of the cluster's CTAs, summed in rank order by everyone
          const double lp = block_sum(llp, red);
          if (DFM_TID == 0) xch[crank] = lp;
          cl_sync(NC);
          double tot = 0.0;
          for (int c = 0; c < NC; ++c) tot += xch[c];
          ll += tot;
          cl_sync(NC);                                     // (xch[0..NC) is reused by the next run)
        } else ll += block_sum(llp, red);
        for (int e = DFM_TID; e < k; e += DFM_NT) zf[e] = zfg[(size_t)(t1 - 1) * k + e];
        DFM_SYNC();
        t = t1 - 1;
        continue;
      }
    }
    if (frozen && !cchg) {
      // ---- frozen step: same Pp, L, S, Tm, Wm, Pf as period last_src; only the means move
      for (int i = DFM_TID; i < k; i += DFM_NT) { double s = 0.0; for (int l = 0; l < k; ++l) s += M[i + k * l] * zf[l]; tv[i] = s; }
      DFM_SYNC();
      for (int e = DFM_TID; e < k; e += DFM_NT) zp[e] = tv[e];
      DFM_SYNC();
      for (int a = DFM_TID; a < r; a += DFM_NT) { double s = bt[a]; for (int c = 0; c < r; ++c) s -= C[a + r * c] * zp[c]; g[a] = s; }
      DFM_SYNC();
      for (int i = DFM_TID; i < k; i += DFM_NT) { double s = zp[i]; for (int a = 0; a < r; ++a) s += Pf[i + k * a] * g[a]; zf[i] = s; }
      DFM_SYNC();
      if (DFM_TID == 0) {
        // quad = q - 2 zp'b + zp'C zp - g'Pff g  with  C zp = b - g  and  Pff g = (zf - zp)[0:r]:  O(r) instead of O(r^2)
        double quad = qt[t];
        for (int a = 0; a < r; ++a) quad += -2.0 * zp[a] * bt[a] + zp[a] * (bt[a] - g[a]) - g[a] * (zf[a] - zp[a]);
        ll += -0.5 * ((double)ntv[t] * DFM_LOG2PI + slr[t] + ldS + quad);
        src[t] = last_src;
      }
      for (int e = DFM_TID; e < k; e += DFM_NT) { zpg[(size_t)t * k + e] = zp[e]; zfg[(size_t)t * k + e] = zf[e]; }
      DFM_SYNC();
      continue;
    }
    frozen = 0;
    if (t == 0) {
      for (int e = DFM_TID; e < kk; e += DFM_NT) Pp[e] = P0[e];
      for (int e = DFM_TID; e < k; e += DFM_NT) zp[e] = 0.0;
      DFM_SYNC();
    } else {
      // P_{t|t-1} = M Pf M' + Q through the companion structure:  AP = M[0:r,:] Pf  (r x k, in Wm), then
      //   [0:r,0:r] = AP M[0:r,:]' + Q,  [0:r, r:] = AP[:, 0:k-r],  [r:, r:] = Pf[0:k-r, 0:k-r]
      for (int e = DFM_TID; e < kk; e += DFM_NT) T3[e] = Pp[e];                 // previous P_{t|t-1}: freeze test below
      wt_gemm(M, 1, k, Pf, k, 1, r, k, k, [&](int a, int j, double v) { Wm[a + r * j] = v; });        // AP = M[0:r,:] Pf
      for (int i = DFM_TID; i < k; i += DFM_NT) { double s = 0.0; for (int l = 0; l < k; ++l) s += M[i + k * l] * zf[l]; tv[i] = s; }
      DFM_SYNC();
      wt_gemm(Wm, 1, r, M, 1, k, r, r, k, [&](int i, int j, double v) { T1[i + k * j] = v + Q[i + r * j]; });   // AP M[0:r,:]' + Q
      for (int e = DFM_TID; e < kk; e += DFM_NT) {
        const int i = e % k, j = e / k;
        if (i < j || i < r) continue;                                           // lower triangle below the top-left block
        T1[e] = (j >= r) ? Pf[(i - r) + k * (j - r)] : Wm[j + r * (i - r)];
      }
      DFM_SYNC();
      // (only the lower triangle was formed; mirror it)
      for (int e = DFM_TID; e < kk; e += DFM_NT) {
        const int i = e % k, j = e / k;
        Pp[e] = (i >= j) ? T1[e] : T1[j + k * i];
      }
      for (int e = DFM_TID; e < k; e += DFM_NT) zp[e] = tv[e];
      DFM_SYNC();
    }
    for (int e = DFM_TID; e < rr; e += DFM_NT) { int i = e % r, j = e / r; L[e] = Pp[i + k * j]; }
    for (int e = DFM_TID; e < rk; e += DFM_NT) { int j = e % k, a = e / k; Tm[e] = Pp[a + k * j]; }       // TmT[j + k a] = Pp[a, j]
    DFM_SYNC();
    bc_chol(L, r, r, dvL, info);                                                // Pff = L L'
    bm_gemm(T4, r, C, r, false, L, r, false, r, r, r, 1.0, 0.0);               // C L
    bm_gemm(S, r, L, r, true, T4, r, false, r, r, r, 1.0, 0.0);                // L' C L
    for (int e = DFM_TID; e < r; e += DFM_NT) S[e + r * e] += 1.0;
    DFM_SYNC();
    bm_symmetrize(S, r, r);
    bc_chol(S, r, r, dvS, info);                                                // S = Ls Ls'
    bt_trsm_lower(L, r, r, dvL, Tm, k, k);                                      // TmT = (L^-1 Pp[0:r,:])'
    for (int e = DFM_TID; e < rk; e += DFM_NT) Wm[e] = Tm[e];
    DFM_SYNC();
    bt_trsm_lower(S, r, r, dvS, Wm, k, k);                                      // WmT = (Ls^-1 Tm)'
    // Pf = Pp - Tm'Tm + Wm'Wm  (both products on the same tile -> lane mapping: an element stays with one thread)
    wt_gemm(Wm, 1, k, Wm, 1, k, k, k, r, [&](int i, int j, double v) { Pf[i + k * j] = Pp[i + k * j] + v; });
    wt_gemm(Tm, 1, k, Tm, 1, k, k, k, r, [&](int i, int j, double v) { Pf[i + k * j] -= v; });
    DFM_SYNC();
    for (int e = DFM_TID; e < kk; e += DFM_NT) { int i = e % k, j = e / k; if (i < j) Pf[e] = Pf[j + k * i]; }
    for (int a = DFM_TID; a < r; a += DFM_NT) { double s = bt[a]; for (int c = 0; c < r; ++c) s -= C[a + r * c] * zp[c]; g[a] = s; }
    DFM_SYNC();
    for (int i = DFM_TID; i < k; i += DFM_NT) { double s = zp[i]; for (int a = 0; a < r; ++a) s += Pf[i + k * a] * g[a]; zf[i] = s; }
    DFM_SYNC();
    if (DFM_TID == 0) {
      ldS = 0.0;
      for (int a = 0; a < r; ++a) ldS -= 2.0 * log(dvS[a]);
      *ldS_sh = ldS;
      double quad = qt[t];             // C zp = b - g and Pff g = (zf - zp)[0:r]: O(r), as in the frozen steps
      for (int a = 0; a < r; ++a) quad += -2.0 * zp[a] * bt[a] + zp[a] * (bt[a] - g[a]) - g[a] * (zf[a] - zp[a]);
      ll += -0.5 * ((double)ntv[t] * DFM_LOG2PI + slr[t] + ldS + quad);
      src[t] = t;
    }
    for (int e = DFM_TID; e < kk; e += DFM_NT) { Ppg[(size_t)t * kk + e] = Pp[e]; Pfg[(size_t)t * kk + e] = Pf[e]; }
    for (int e = DFM_TID; e < k; e += DFM_NT) { zpg[(size_t)t * k + e] = zp[e]; zfg[(size_t)t * k + e] = zf[e]; }
    last_src = t;
    if (t >= 1 && !cchg) {                                                      // steady state reached?  (T3 = previous Pp)
      double dm = 0.0, pm = 0.0;
      for (int e = DFM_TID; e < kk; e += DFM_NT) { dm = fmax(dm, fabs(Pp[e] - T3[e])); pm = fmax(pm, fabs(Pp[e])); }
      block_max2(dm, pm, red2);
      frozen = (dm <= 1e-14 * pm) ? 1 : 0;
    }
    DFM_SYNC();
  }
  // ------------------------------------------------------------------ backward: RTS smoother
  for (int e = DFM_TID; e < kk; e += DFM_NT) Psn[e] = Pf[e];
  for (int e = DFM_TID; e < k; e += DFM_NT) zsn[e] = zf[e];
  DFM_SYNC();
  for (int e = DFM_TID; e < r; e += DFM_NT) Fs[(T - 1) + (size_t)T * e] = zsn[e];
  for (int e = DFM_TID; e < rr; e += DFM_NT) {
    int a = e % r, c = e / r;
    if (psf && a >= c) PsF[(T - 1) + (size_t)T * pidx(a, c)] = Psn[a + k * c];
    SffA[e] = zsn[a] * zsn[c] + Psn[a + k * c];
  }
  DFM_SYNC();
  int jpp = -1, jpf = -1, ps_frozen = 0;           // periods whose covariances built the gain J in T3; smoothed covariance frozen?
  int brun_known = T;                              // backward runs: no search above this period (a shorter run is in progress)
  for (int t = T - 2; t >= 0; --t) {
    const int sp = src[t + 1], sf = src[t];
    const bool newJ = (sp != jpp) || (sf != jpf);
    if (newJ) ps_frozen = 0;
    if (!newJ && ps_frozen && jpp == jpf && t <= brun_known) {
      // ---- frozen backward run: every period down to tl uses the gain in T3 and the smoothed covariance in Ps
      if (DFM_TID == 0) info[1] = -1;
      DFM_SYNC();
      for (int base_ = t - 1; base_ >= 0; base_ -= DFM_NT) {
        const int tp = base_ - DFM_TID;
        if (tp >= 0 && src[tp] != jpf) atomicMax(&info[1], tp);
        DFM_SYNC();
        const int v = info[1];
        DFM_SYNC();
        if (v >= 0) break;
      }
      const int tl = info[1] + 1, Lr = t - tl + 1;
      brun_known = tl - 1;
      if (Lr >= EM_RUN_MIN) {
        // zs_t = J zs_{t+1} + v_t,  v_t = zf_t - J zp_{t+1}   (J is in T3)
        const int lds = em_lds(k);
        double* Zq = stg;                              // [TT][lds]      zp_{t0+1} .. zp_{t0+len}
        for (int t0 = tl, ti = 0; t0 <= t; t0 += TT, ++ti) {
          if (ti % NC != crank) continue;
          const int len = (t - t0 + 1 < TT) ? t - t0 + 1 : TT;
          DFM_SYNC();
          {
            const double* g0 = zpg + (size_t)(t0 + 1) * k;
#pragma unroll 4
            for (int e = DFM_TID; e < len * k; e += DFM_NT) { const int tt = e / k, i = e - tt * k; Zq[tt * lds + i] = g0[e]; }
          }
          DFM_SYNC();
          wt_gemm(Zq, lds, 1, T3, 1, k, len, k, k, [&](int m, int n, double v) { zfg[(size_t)(t0 + m) * k + n] -= v; });
        }
        DFM_SYNC();
        cl_sync(NC);
        em_run_scan(zfg, k, t, Lr, -1, T3, zsn, T1, Pf, T2, wb, stg, stg_doubles, NC, crank, xbnd);   // (T1, Pf, T2 are free here; zfg now holds zs_t)
        cl_sync(NC);
        // Gram sums of the smoothed means: S00 (k x k), S11 (r x k) as DMMA products over tiles of zs rows staged in shared
        // memory; a warp's output tiles stay in registers over the tiles of the run
        const double cnt = (double)Lr;
        const int nt00 = ((k + 7) >> 3) * ((k + 7) >> 3), nt11 = ((r + 7) >> 3) * ((k + 7) >> 3);
        double acc[EM_TQ][2];
#pragma unroll
        for (int q = 0; q < EM_TQ; ++q) { acc[q][0] = 0.0; acc[q][1] = 0.0; }
#ifndef DFM_EMU
        const bool in_regs = nt00 + nt11 <= EM_TQ * DFM_NWARP;
#else
        const bool in_regs = false;
#endif
        const int NCg = in_regs ? NC : 1, crg = in_regs ? crank : 0;      // (the plain-sum path is not split over the cluster)
        double* Zs = stg;                              // [TT + 1][lds]   zs_{t0} .. zs_{t0+len}
        for (int t0 = tl, ti = 0; t0 <= t; t0 += TT, ++ti) {
          if (ti % NCg != crg) continue;
          const int len = (t - t0 + 1 < TT) ? t - t0 + 1 : TT;
          DFM_SYNC();
          {
            const double* g0 = zfg + (size_t)t0 * k;
#pragma unroll 4
            for (int e = DFM_TID; e < (len + 1) * k; e += DFM_NT) {
              const int tt = e / k, i = e - tt * k;
              Zs[tt * lds + i] = (t0 + tt > t) ? zsn[i] : g0[e];
            }
          }
          DFM_SYNC();
          for (int e = DFM_TID; e < r * len; e += DFM_NT) { const int a = e / len, tt = e - a * len; Fs[t0 + tt + (size_t)T * a] = Zs[tt * lds + a]; }
          if (in_regs) {
            wt_gemm_acc(Zs, 1, lds, Zs, 1, lds, k, k, len, 0, acc);                    // sum_t zs_t zs_t'
            wt_gemm_acc(Zs + lds, 1, lds, Zs, 1, lds, r, k, len, nt00, acc);           // sum_t zs_{t+1}[0:r] zs_t'
          } else {
            for (int e = DFM_TID; e < kk + rk; e += DFM_NT) {                   // (emulation / very large k: plain sums)
              double g0 = 0.0;
              if (e < kk) {
                const int i = e % k, j = e / k;
                for (int tt = 0; tt < len; ++tt) g0 += Zs[tt * lds + i] * Zs[tt * lds + j];
                S00[e] += g0;
                if (i < r && j < r) { SffA[i + r * j] += g0; Sff2[i + r * j] += g0; }
              } else { const int e2 = e - kk, i = e2 % r, j = e2 / r; for (int tt = 0; tt < len; ++tt) g0 += Zs[(tt + 1) * lds + i] * Zs[tt * lds + j]; S11[e2] += g0; }
            }
          }
        }
        DFM_SYNC();
        // zs_tl (k) -> tv for the Sff2 correction; fold the register sums into the shared accumulators
        for (int e = DFM_TID; e < k; e += DFM_NT) tv[e] = zfg[(size_t)tl * k + e];
        if (in_regs && NC > 1) {
          // partial Gram sums of the cluster's CTAs through global memory, added in rank order by everyone
          double* mine = xgram + (size_t)crank * (kk + rk);
          wt_acc_visit(k, k, 0, acc, [&](int i, int j, double v) { mine[i + k * j] = v; });
          wt_acc_visit(r, k, nt00, acc, [&](int i, int j, double v) { mine[kk + i + r * j] = v; });
          DFM_SYNC();
          cl_sync(NC);
          for (int e = DFM_TID; e < kk + rk; e += DFM_NT) {
            double v = 0.0;
            for (int c = 0; c < NC; ++c) v += xgram[(size_t)c * (kk + rk) + e];
            if (e < kk) {
              S00[e] += v;
              const int i = e % k, j = e / k;
              if (i < r && j < r) { SffA[i + r * j] += v; Sff2[i + r * j] += v; }
            } else S11[e - kk] += v;
          }
        } else if (in_regs) {
          wt_acc_visit(k, k, 0, acc, [&](int i, int j, double v) {
            S00[i + k * j] += v;
            if (i < r && j < r) { SffA[i + r * j] += v; Sff2[i + r * j] += v; }            // r x r block of the same Gram sum
          });
          wt_acc_visit(r, k, nt00, acc, [&](int i, int j, double v) { S11[i + r * j] += v; });
        }
        DFM_SYNC();
        for (int e = DFM_TID; e < rr; e += DFM_NT) {                            // (zsn: still the state that entered the run)
          const int i = e % r, j = e / r;
          SffA[e] += cnt * Ps[i + k * j];
          Sff2[e] += cnt * Ps[i + k * j] - tv[i] * tv[j] + zsn[i] * zsn[j];
        }
        for (int e = DFM_TID; e < kk; e += DFM_NT) S00[e] += cnt * Ps[e];
        for (int e = DFM_TID; e < rk; e += DFM_NT) S11[e] += cnt * Tm[e];
        if (psf) for (int a = 0, pe = 0; a < r; ++a)
          for (int c = 0; c <= a; ++c, ++pe) {
            const double v = Ps[a + k * c];
            double* dst = PsF + (size_t)T * pe;
            for (int tt = tl + DFM_TID; tt <= t; tt += DFM_NT) dst[tt] = v;
          }
        DFM_SYNC();
        for (int e = DFM_TID; e < k; e += DFM_NT) zsn[e] = tv[e];
        DFM_SYNC();
        t = tl;
        continue;
      }
    }
    for (int e = DFM_TID; e < k; e += DFM_NT) { zp[e] = zpg[(size_t)(t + 1) * k + e]; zf[e] = zfg[(size_t)t * k + e]; }
    if (!ps_frozen) for (int e = DFM_TID; e < kk; e += DFM_NT) { T1[e] = Ppg[(size_t)sp * kk + e]; Pf[e] = Pfg[(size_t)sf * kk + e]; }
    DFM_SYNC();
    if (newJ) {
      // J = Pf M' Pp^-1, row by row:  T3 <- Pf M' (companion structure: columns >= r are a shift of Pf), T2 = chol(Pp) on
      // warp 0 meanwhile, then  L y = x, L' z = y  on the rows of T3 (thread per row)
      for (int e = DFM_TID; e < kk; e += DFM_NT) {
        T2[e] = T1[e];
        const int i = e % k, j = e / k;
        if (j >= r) T3[e] = Pf[i + k * (j - r)];
      }
      wt_gemm(Pf, 1, k, M, 1, k, k, r, k, [&](int i, int j, double v) { T3[i + k * j] = v; });
      DFM_SYNC();
      bc_chol(T2, k, k, dvL, info);
      // J = (Pf M') Pp^-1 = (Pf M') U U',  U = L^-T:  U' = L^-1 by forward substitution on the rows of the identity (thread per
      // row, registers), then two tensor-core products -- the back substitution, whose row stays in shared memory, cost
      // 16 K cycles at k = 32
      for (int e = DFM_TID; e < kk; e += DFM_NT) { const int j = e % k, a = e / k; Pp[e] = (j == a) ? 1.0 : 0.0; }
      DFM_SYNC();
      bt_trsm_lower(T2, k, k, dvL, Pp, k, k);                                   // Pp[j + k a] = (L^-1)[a, j]  (= U[j, a])
      wt_gemm(T3, 1, k, Pp, k, 1, k, k, k, [&](int i, int j, double v) { T2[i + k * j] = v; });      // (Pf M') U
      DFM_SYNC();
      wt_gemm(T2, 1, k, Pp, 1, k, k, k, k, [&](int i, int j, double v) { T3[i + k * j] = v; });      // ... U' = J
      DFM_SYNC();
      jpp = sp; jpf = sf;
    }
    for (int e = DFM_TID; e < k; e += DFM_NT) dv[e] = zsn[e] - zp[e];
    if (!ps_frozen) for (int e = DFM_TID; e < kk; e += DFM_NT) T1[e] = Psn[e] - T1[e];     // D = Ps(t+1) - Pp(t+1)
    DFM_SYNC();
    for (int i = DFM_TID; i < k; i += DFM_NT) { double s = zf[i]; for (int l = 0; l < k; ++l) s += T3[i + k * l] * dv[l]; zs[i] = s; }
    if (!ps_frozen) {
      wt_gemm(T3, 1, k, T1, k, 1, k, k, k, [&](int i, int j, double v) { T2[i + k * j] = v; });           // J D
      wt_gemm(Psn, 1, k, T3, 1, k, r, k, k, [&](int i, int j, double v) { Tm[i + r * j] = v; });          // Pc[0:r,:] = Ps(t+1)[0:r,:] J'
      DFM_SYNC();
      wt_gemm(T2, 1, k, T3, 1, k, k, k, k, [&](int i, int j, double v) { Ps[i + k * j] = Pf[i + k * j] + v; });   // Pf + (J D) J'
      DFM_SYNC();
      bm_symmetrize(Ps, k, k);
      if (!newJ) {                                                              // smoothed covariance at its steady state?
        double dm = 0.0, pm = 0.0;
        for (int e = DFM_TID; e < kk; e += DFM_NT) { dm = fmax(dm, fabs(Ps[e] - Psn[e])); pm = fmax(pm, fabs(Ps[e])); }
        block_max2(dm, pm, red2);
        ps_frozen = (dm <= 1e-14 * pm) ? 1 : 0;      // from the next period on: Ps = Psn, Tm as they are
      }
    } else DFM_SYNC();
    for (int e = DFM_TID; e < rk; e += DFM_NT) { int i = e % r, j = e / r; S11[e] += zsn[i] * zs[j] + Tm[e]; }
    for (int e = DFM_TID; e < kk; e += DFM_NT) { int i = e % k, j = e / k; S00[e] += zs[i] * zs[j] + Ps[e]; }
    for (int e = DFM_TID; e < rr; e += DFM_NT) {
      int a = e % r, c = e / r;
      Sff2[e] += zsn[a] * zsn[c] + Psn[a + k * c];
      SffA[e] += zs[a] * zs[c] + Ps[a + k * c];
      if (psf && a >= c) PsF[t + (size_t)T * pidx(a, c)] = Ps[a + k * c];
    }
    for (int e = DFM_TID; e < r; e += DFM_NT) Fs[t + (size_t)T * e] = zs[e];
    DFM_SYNC();
    for (int e = DFM_TID; e < kk; e += DFM_NT) Psn[e] = Ps[e];
    for (int e = DFM_TID; e < k; e += DFM_NT) zsn[e] = zs[e];
    DFM_SYNC();
  }
  // ------------------------------------------------------------------ transition M-step
  // A = S11 S00^-1 (row by row: S00 A[i,:]' = S11[i,:]') ;  Q = (Sff2 - A S11') / (T-1)
  bm_copy(T2, k, S00, k, k, k);
  bc_chol(T2, k, k, dvL, info);
  for (int e = DFM_TID; e < rk; e += DFM_NT) Wm[e] = S11[e];
  DFM_SYNC();
  bt_trsm_lower(T2, k, k, dvL, Wm, r, r);
  bt_trsm_lowerT(T2, k, k, dvL, Wm, r, r);                                           // Wm = A (r x k)
  for (int e = DFM_TID; e < rr; e += DFM_NT) {
    int a = e % r, c = e / r;
    double s = Sff2[e];
    for (int l = 0; l < k; ++l) s -= Wm[a + r * l] * S11[c + r * l];           // (A S11')[a,c]
    T4[e] = s / (double)(T - 1);
  }
  DFM_SYNC();
  bm_symmetrize(T4, r, r);
  for (int e = DFM_TID; e < rk; e += DFM_NT) Anew_[(size_t)b * rk + e] = Wm[e];
  for (int e = DFM_TID; e < rr; e += DFM_NT) { Qnew_[(size_t)b * rr + e] = T4[e]; SffAll_[(size_t)b * rr + e] = SffA[e]; }
  if (DFM_TID == 0 && crank == 0) {                  // (one CTA of the cluster updates the panel's state: the update is not idempotent)
    int it = st[b].iters;
    loglik_[(size_t)b * max_iter + it] = ll;
    st[b].ll_prev = st[b].ll; st[b].ll = ll;
    if (it >= 1 && fabs(ll - st[b].ll_prev) <= tol * 0.5 * (fabs(ll) + fabs(st[b].ll_prev))) st[b].conv_pending = 1;
    if (*info || !(ll == ll)) st[b].status = 3;
  }
}

// Linear restrictions on the loadings (LambdaConstraint, standardized units), uploaded once per call as a per-series CSR:
// the rows of series i are off[i] .. off[i+1]-1, row q is H[q*r .. q*r+r) (row-major) with value h[q].  off == nullptr: none.
struct EmConstr { const int* off; const double* H; const double* h; };
#define EM_CONSTR_PIVOT_RTOL 1e-12     // G pivot <= this * G_jj: dependent restriction rows

// shared scratch of lam_constr_correct (doubles): Y r x r, G packed, d r
__host__ __device__ inline int em_constr_scratch(int r) { return r * r + r * (r + 1) / 2 + r; }

// Restricted M-step of one series, one thread:  lam (in: lu = S^-1 s, out: lu - Y G^-1 (H lu - h)) with Y = S^-1 H',
// G = H Y; solve(v) overwrites v (r) with S^-1 v using the caller's Cholesky factor of S.  m rows, m <= r.
// ws: em_constr_scratch(r) doubles.  Returns 1 when G is singular (lam unchanged then).
template <class Solve>
__device__ inline int lam_constr_correct(double* lam, int r, const double* H, const double* h, int m, double* ws, Solve solve) {
  double* Y = ws; double* G = Y + r * r; double* d = G + r * (r + 1) / 2;
  for (int j = 0; j < m; ++j) {
    const double* hj = H + (size_t)j * r;
    for (int a = 0; a < r; ++a) Y[a + r * j] = hj[a];
    solve(Y + r * j);
    double v = -h[j];
    for (int a = 0; a < r; ++a) v += hj[a] * lam[a];
    d[j] = v;
    for (int l = 0; l <= j; ++l) { double g = 0.0; for (int a = 0; a < r; ++a) g += hj[a] * Y[a + r * l]; G[pidx(j, l)] = g; }
  }
  for (int j = 0; j < m; ++j) {                       // packed Cholesky of G with a relative pivot test
    double p = G[pidx(j, j)];
    const double g0 = p;
    for (int c = 0; c < j; ++c) p -= G[pidx(j, c)] * G[pidx(j, c)];
    if (!(p > EM_CONSTR_PIVOT_RTOL * g0)) return 1;
    p = sqrt(p);
    G[pidx(j, j)] = p;
    for (int i = j + 1; i < m; ++i) {
      double s = G[pidx(i, j)];
      for (int c = 0; c < j; ++c) s -= G[pidx(i, c)] * G[pidx(j, c)];
      G[pidx(i, j)] = s / p;
    }
  }
  chol_resolve_packed(G, d, m, 1);
  for (int a = 0; a < r; ++a) { double v = lam[a]; for (int j = 0; j < m; ++j) v -= Y[a + r * j] * d[j]; lam[a] = v; }
  return 0;
}

// Measurement M-step: one block per series.  S_ff^(i) = SffAll - sum_{t missing} E_t.
// Lam_i = S_ff^(i)^-1 S_xf^(i);  R_i = (S_xx - 2 lam'S_xf + lam' S_ff lam) / T_i.   grid (N, B).
// With restrictions (cs.off != nullptr) a restricted series' Lam_i is corrected (lam_constr_correct) with the packed Cholesky
// factor of S_ff^(i) before R_i is formed; shared memory then holds em_constr_scratch(r) more doubles.
__global__ void k_em_mstep_series(const double* __restrict__ Xall, const double* __restrict__ Fs_,
                                  const double* __restrict__ PsF_, const double* __restrict__ SffAll_, int T, int N,
                                  int r, double* __restrict__ LamAll, double* __restrict__ Rall, EmState* st, int skip_bal,
                                  EmConstr cs) {
  DFM_SMEM(sm);
  int i = DFM_BX, b = DFM_BY;
  if (st[b].done) return;
  if (skip_bal && !st[b].has_missing) return;                 // balanced panels: k_emb_mstep
  int np = r * (r + 1) / 2;
  double* Lam = LamAll + (size_t)b * N * r; double* R = Rall + (size_t)b * N;
  if (is_nan(Lam[i]) || is_nan(R[i])) return;         // excluded series stay excluded
  const double* x = Xall + ((size_t)b * N + i) * T;
  const double* Fs = Fs_ + (size_t)b * T * r; const double* PsF = PsF_ + (size_t)b * T * np;
  const double* SffA = SffAll_ + (size_t)b * r * r;
  double* A = sm; double* c = A + np; double* sc = c + r; double* A0 = sc + 4;
  int hm = st[b].has_missing;
  int nwork = np + r + 2;
  for (int e = DFM_TID; e < nwork; e += DFM_NT) {
    double s = 0.0;
    if (e < np) {
      int a = 0; while ((a + 1) * (a + 2) / 2 <= e) ++a;
      int cc = e - a * (a + 1) / 2;
      if (hm) for (int t = 0; t < T; ++t) if (is_nan(x[t])) s += Fs[t + (size_t)T * a] * Fs[t + (size_t)T * cc] + PsF[t + (size_t)T * e];
      A[e] = SffA[a + r * cc] - s; A0[e] = A[e];
    } else if (e < np + r) {
      const double* fa = Fs + (size_t)T * (e - np);
      for (int t = 0; t < T; ++t) { double v = x[t]; if (!is_nan(v)) s += v * fa[t]; }
      c[e - np] = s;
    } else if (e == np + r) { for (int t = 0; t < T; ++t) if (!is_nan(x[t])) s += 1.0; sc[0] = s; }
    else { for (int t = 0; t < T; ++t) { double v = x[t]; if (!is_nan(v)) s += v * v; } sc[1] = s; }
  }
  DFM_SYNC();
  if (DFM_TID != 0) return;
  if (sc[0] < 1.0) return;
  double sxf[64];
  for (int a = 0; a < r; ++a) sxf[a] = c[a];
  if (chol_solve_packed(A, c, r, 1)) { st[b].status = 3; return; }
  if (cs.off) {
    const int q0 = cs.off[i], m = cs.off[i + 1] - q0;
    if (m > 0 && lam_constr_correct(c, r, cs.H + (size_t)q0 * r, cs.h + q0, m, A0 + np,
                                    [&](double* v) { chol_resolve_packed(A, v, r, 1); })) { st[b].status = 3; return; }
  }
  double q1 = 0.0, q2 = 0.0;
  for (int a = 0; a < r; ++a) {
    q1 += c[a] * sxf[a];
    for (int cc = 0; cc < r; ++cc) q2 += c[a] * c[cc] * ((a >= cc) ? A0[pidx(a, cc)] : A0[pidx(cc, a)]);
  }
  for (int a = 0; a < r; ++a) Lam[i + (size_t)N * a] = c[a];
  R[i] = (sc[1] - 2.0 * q1 + q2) / sc[0];
}

// unpack PsF (packed, [T x np]) to r x r x T column-major for the API output.
__global__ void k_unpack_psf(const double* __restrict__ PsF_, int T, int r, double* __restrict__ out) {
  int b = DFM_BY, np = r * (r + 1) / 2;
  const double* PsF = PsF_ + (size_t)b * T * np;
  double* o = out + (size_t)b * T * r * r;
  for (long long e = (long long)DFM_BX * DFM_NT + DFM_TID; e < (long long)T * r * r; e += (long long)DFM_GX * DFM_NT) {
    int a = (int)(e % r), c = (int)((e / r) % r), t = (int)(e / ((long long)r * r));
    o[e] = (a >= c) ? PsF[t + (size_t)T * pidx(a, c)] : PsF[t + (size_t)T * pidx(c, a)];
  }
}

__global__ void k_em_count_active(const EmState* st, int B, int* out) {
  DFM_SMEM(sm);
  double n = 0.0;
  for (int b = DFM_TID; b < B; b += DFM_NT) n += st[b].done ? 0.0 : 1.0;
  n = block_sum(n, sm);
  if (DFM_TID == 0) *out = (int)n;
}

__global__ void k_em_count_missing(const EmState* st, int B, int* out) {
  DFM_SMEM(sm);
  double n = 0.0;
  for (int b = DFM_TID; b < B; b += DFM_NT) n += st[b].has_missing ? 1.0 : 0.0;
  n = block_sum(n, sm);
  if (DFM_TID == 0) *out = (int)n;
}

__global__ void k_em_collect(const EmState* st, int* iters, int* status) {
  if (DFM_TID != 0) return;
  int b = DFM_BX;
  iters[b] = st[b].iters; status[b] = st[b].status;
}

__global__ void k_fill(double* p, long long n, double v) {
  for (long long e = (long long)DFM_BX * DFM_NT + DFM_TID; e < n; e += (long long)DFM_GX * DFM_NT) p[e] = v;
}

}  // namespace dfm
