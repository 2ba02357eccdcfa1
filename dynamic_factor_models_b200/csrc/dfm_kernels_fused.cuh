// dfm_kernels_fused.cuh -- FUSED per-panel EM kernel: the whole EM loop (E-step Kalman filter + RTS
// smoother, M-step) of one panel runs inside one CTA; one launch covers all panels and all
// iterations.  Row a' of SURVEY.md section 8, fast path for p = 1, r <= 8, balanced panels (k = r).
//
//  * panel reads: exactly two streaming passes per EM iteration (E-step contraction
//    b_t = Lam' R^-1 x_t and M-step contraction S_xf = X' E[f]), straight from HBM into FP64
//    tensor-core fragments: mma.sync.m8n8k4.f64 (SASS DMMA.8x8x4) -- wgmma has no FP64 kind and
//    the 1e-5 parity bar needs FP64 (DESIGN.md);
//  * Lam, 1/R and the T x r state buffer Z (b_t -> f_t|t -> f_t|T in place) live in shared memory;
//  * the covariance recursion of a balanced panel is data independent and time invariant: warp 0
//    runs it explicitly only until P_{t|t-1} stops changing (relative 1e-14; a handful of steps at
//    N = 200), forward and backward, and closes the moment sums in closed form over the frozen
//    range (validated in tools/proto_fused.py against the oracle);
//  * the mean recursions are two T-step r x r matvec chains on r lanes of warp 0.
// The serial logic is written phase-style (loops over DFM_LANE + DFM_WSYNC) so that the host
// emulation harness (tests/emu) executes the very same source; only the two DMMA loops have an
// #ifdef DFM_EMU plain-loop twin.
#pragma once
#include "dfm_common.cuh"

namespace dfm {

#define FZ 8   // number of state components kept in Z (= DMMA tile width)
// Z and Lam are stored COMPONENT-major with a leading dimension == 4 (mod 16) doubles: conflict-free
// for thread-per-period row access, for the 8-lane recursion groups and (per half-warp) for the DMMA
// B-fragments.
#define ZI(t_, i_) ((i_) * Tp + (t_))
#define LI(n_, c_) ((c_) * Np + (n_))
__host__ __device__ inline int pad4mod16(int x) { return x + ((4 - x % 16) + 16) % 16; }

struct FusedArgs {
  const double* X;      // [B][N][T] column-major panels
  double* Lam;          // [B][N*r] column-major (in: init, out: final)
  double* R;            // [B][N]
  double* A;            // [B][r*r] column-major
  double* Q;            // [B][r*r]
  const double* P0;     // [B][r*r]
  double* Fs;           // [B][T*r] column-major  (out)
  double* PsF;          // [B][T*np] packed        (out)
  double* loglik;       // [B][max_iter]           (pre-filled with NaN)
  int* iters; int* status;
  double* scratch;      // [gridDim.x][T * FUSED_SCR]
  int B, T, N, max_iter;
  double tol;
  // streaming host path (k_em_fused2 only): the kernel is launched BEFORE the panels are on the device; ready[c] is
  // set (by a stream-ordered 4-byte H2D copy that follows chunk c's data on the copy stream) once panels
  // [c * ready_chunk, (c+1) * ready_chunk) and their initial parameters have arrived.  NULL = everything resident.
  const int* ready; int ready_chunk;
  int* done;                 // streaming host path: done[b] = 1 (mapped pinned host memory) once panel b's results are in device memory
  double* P0out;             // non-NULL: compute P0 in the kernel (Lyapunov doubling of (A, Q), p0_steps steps, as k_lyapunov)
  int p0_steps;              //           and store it here ([B][r*r]).  With ready or P0out set the kernel also pre-fills its loglik rows.
  int l2_win[2];             // k_em_fused2: turn window per panel pass (copies): full rounds, tail round (f2_round_win)
};
#define FUSED_SCR(R_) (5 * (R_) * (R_) + 1)

__device__ __forceinline__ double w_max(double v) {
#ifndef DFM_EMU
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
#endif
  return v;
}

// ---- warp-0 small dense ops on row-major R x R matrices in shared memory ------------------------
// NOT inlined on the GPU: the chain calls them ~100 times per EM iteration; inlined + unrolled they
// made one chain step ~40 KB of straight-line code executed by a single warp, i.e. instruction-cache
// misses all the way.
#ifdef DFM_EMU
#define DFM_HELPER inline
#else
#define DFM_HELPER __device__ __noinline__
#endif
template <int R>
DFM_HELPER void w_gemm(double* C, const double* A, bool ta, const double* B, bool tb) {
#ifndef DFM_EMU
  if (R == 8) {
    // 8x8x8 product on the FP64 tensor path: two DMMA.8x8x4 with fragments straight from shared memory
    const int lane = threadIdx.x & 31, lr = lane >> 2, lc = lane & 3;
    double d0 = 0.0, d1 = 0.0;
#pragma unroll
    for (int kc = 0; kc < 2; ++kc) {
      const int kk = 4 * kc + lc;
      const double av = ta ? A[kk * 8 + lr] : A[lr * 8 + kk];      // A-fragment: op(A)[lr][kk]
      const double bv = tb ? B[lr * 8 + kk] : B[kk * 8 + lr];      // B-fragment: op(B)[kk][lr]
      asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
                   : "+d"(d0), "+d"(d1) : "d"(av), "d"(bv));
    }
    C[lr * 8 + 2 * lc] = d0; C[lr * 8 + 2 * lc + 1] = d1;
    __syncwarp();
    return;
  }
#endif
  for (int e = DFM_LANE; e < R * R; e += DFM_WSZ) {
    int i = e / R, j = e % R;
    double s = 0.0;
#pragma unroll
    for (int l = 0; l < R; ++l) s += (ta ? A[l * R + i] : A[i * R + l]) * (tb ? B[j * R + l] : B[l * R + j]);
    C[e] = s;
  }
  DFM_WSYNC();
}
template <int R>
DFM_HELPER void w_sym(double* A) {
#ifndef DFM_EMU
  if (R == 8) {                 // every lane: read its two elements and their transposes, then write
    const int lane = threadIdx.x & 31, i = lane >> 2, j0 = 2 * (lane & 3);
    const double v0 = 0.5 * (A[i * 8 + j0] + A[j0 * 8 + i]), v1 = 0.5 * (A[i * 8 + j0 + 1] + A[(j0 + 1) * 8 + i]);
    __syncwarp();
    A[i * 8 + j0] = v0; A[i * 8 + j0 + 1] = v1;
    __syncwarp();
    return;
  }
#endif
  for (int e = DFM_LANE; e < R * R; e += DFM_WSZ) {
    int i = e / R, j = e % R;
    if (i > j) { double v = 0.5 * (A[i * R + j] + A[j * R + i]); A[i * R + j] = v; A[j * R + i] = v; }
  }
  DFM_WSYNC();
}
// Gauss-Jordan inverse (no pivoting; SPD input) + log det.  Ai <- A^-1.  tmp: 2R doubles.
template <int R>
DFM_HELPER double w_inv(double* Ai, const double* A, double* tmp, int* bad) {
#ifndef DFM_EMU
  if (R == 8) {
    // register version: lane owns elements (i, j0) and (i, j0+1), i = lane/4, j0 = 2 (lane%4); per
    // pivot four double shuffles (pivot, its row for my columns, its column for my row) -- no shared
    // memory round trips, faster than the generic version below (tools/bench_chain.cu)
    const int lane = threadIdx.x & 31, i = lane >> 2, q = lane & 3, j0 = 2 * q;
    double x0 = A[i * 8 + j0], x1 = A[i * 8 + j0 + 1];
    double pp = 1.0;
#pragma unroll
    for (int p = 0; p < 8; ++p) {
      const double sel = (p & 1) ? x1 : x0;                               // my element in column-pair slot p&1
      double piv = __shfl_sync(0xffffffffu, sel, p * 4 + (p >> 1));       // a[p][p]
      const double rp0 = __shfl_sync(0xffffffffu, x0, p * 4 + q);         // a[p][j0]
      const double rp1 = __shfl_sync(0xffffffffu, x1, p * 4 + q);         // a[p][j0+1]
      const double cp = __shfl_sync(0xffffffffu, sel, (lane & ~3) + (p >> 1));   // a[i][p]
      if (!(piv > 0.0)) { *bad = 1; piv = 1.0; }
      pp *= piv;
      const double d = 1.0 / piv, cd = cp * d;
      const bool ip = (i == p);
      x0 = ip ? ((j0 == p) ? d : rp0 * d) : ((j0 == p) ? -cd : x0 - cd * rp0);
      x1 = ip ? ((j0 + 1 == p) ? d : rp1 * d) : ((j0 + 1 == p) ? -cd : x1 - cd * rp1);
    }
    Ai[i * 8 + j0] = x0; Ai[i * 8 + j0 + 1] = x1;
    __syncwarp();
    (void)tmp;
    return log(pp);
  }
#endif
  for (int e = DFM_LANE; e < R * R; e += DFM_WSZ) Ai[e] = A[e];
  DFM_WSYNC();
  double pp = 1.0;
  for (int p = 0; p < R; ++p) {
    for (int e = DFM_LANE; e < R; e += DFM_WSZ) { tmp[e] = Ai[p * R + e]; tmp[R + e] = Ai[e * R + p]; }
    DFM_WSYNC();
    double piv = tmp[p];
    if (!(piv > 0.0)) { *bad = 1; piv = 1.0; }
    pp *= piv;                              // det = product of pivots (R <= 8: no over/underflow concern)
    double d = 1.0 / piv;
    for (int e = DFM_LANE; e < R * R; e += DFM_WSZ) {
      int i = e / R, j = e % R;
      double v;
      if (i == p && j == p) v = d;
      else if (i == p) v = tmp[j] * d;
      else if (j == p) v = -tmp[R + i] * d;
      else v = Ai[e] - tmp[R + i] * tmp[j] * d;
      Ai[e] = v;
    }
    DFM_WSYNC();
  }
  return log(pp);
}

// chunk length of the parallel-in-time scan for n steps on ng 8-lane groups: odd (the 4 groups of a warp then hit
// different banks) and at most ng chunks
__device__ __forceinline__ int blk_chunk_len(int n, int ng) {
  int Lc = (n + ng - 1) / ng;
  if (Lc > 1 && !(Lc & 1)) Lc += 1;
  return Lc;
}

// pw <- Cf^ex by binary exponentiation (one warp; base, pw2: R*R scratch each)
template <int R>
__device__ __forceinline__ void w_matpow(double* pw, const double* Cf, int ex0, double* base, double* pw2) {
  for (int e = DFM_LANE; e < R * R; e += DFM_WSZ) { int i = e / R, j = e % R; pw[e] = (i == j) ? 1.0 : 0.0; base[e] = Cf[e]; }
  DFM_WSYNC();
  for (int ex = ex0; ex > 0; ex >>= 1) {
    if (ex & 1) { w_gemm<R>(pw2, pw, false, base, false); for (int e = DFM_LANE; e < R * R; e += DFM_WSZ) pw[e] = pw2[e]; DFM_WSYNC(); }
    if (ex > 1) { w_gemm<R>(pw2, base, false, base, false); for (int e = DFM_LANE; e < R * R; e += DFM_WSZ) base[e] = pw2[e]; DFM_WSYNC(); }
  }
}

// Constant-coefficient linear recursion  Z[t] <- Cf Z[t - dir] + Z[t],  t = t0, t0+dir, ... (n steps),
// parallel in time over nthr threads of the CTA: the n steps are cut into chunks of Lc = blk_chunk_len(n, nthr/8)
// owned by 8-lane groups (lane = state component, coefficient row in registers);
//   pass 1  every chunk runs the recursion from a zero state (chunk 0 from the true state),
//   bound   one group propagates the true chunk-end states with Cf^Lc (pw, by repeated squaring),
//   pass 2  every chunk adds Cf^(s+1) * (true state entering the chunk).
// Exact up to rounding (linear recurrence).  Called by ALL threads; ends with a block barrier.
// smem: pw, pw2 [R*R], bnd [(3 ng + 1) R + R R].  pw_ready: pw already holds Cf^Lc (computed elsewhere, e.g. by the
// chain warp of k_em_fused2 while the panel streams); otherwise warp 0 computes it here.  pl1..pl4 (optional, GPU):
// pw^2, pw^4, pw^8, pw^16 -- the boundary propagation is then a Kogge-Stone scan over the chunks (5 levels, all groups
// in parallel) instead of nch - 1 serial matrix-vector steps.
template <int R>
__device__ __forceinline__ void blk_recur(double* Z, int Tp, const double* Cf, double* pw, double* pw2, double* bnd, int t0, int n, int dir, int nthr,
                                          bool pw_ready = false, const double* pl1 = nullptr, const double* pl2 = nullptr,
                                          const double* pl3 = nullptr, const double* pl4 = nullptr) {
  if (n <= 0) return;
  // nthr = number of threads taking part (threads 0 .. nthr-1 of the CTA, a multiple of 32); they synchronise
  // on named barrier 2, so the remaining warps of the CTA may do something else meanwhile
  const int ng = nthr / 8;
#ifndef DFM_EMU
#define BLK_SYNC() asm volatile("bar.sync 2, %0;" ::"r"(nthr) : "memory")
#else
#define BLK_SYNC() ((void)0)
#endif
  // ng = number of 8-lane groups of the CTA (blockDim / 8).  chunk length: odd (=> the 4 groups of a
  // warp hit different banks) and at most ng chunks.  bnd: [(3 ng + 1) R + R R] doubles.
  const int Lc = blk_chunk_len(n, ng);
  const int nch = (n + Lc - 1) / Lc;
  if (DFM_WARP == 0 && nch > 1 && !pw_ready) w_matpow<R>(pw, Cf, Lc, bnd + (size_t)(3 * ng + 1) * R, pw2);   // scratch beyond the boundary vectors
  // ---- pass 1
#ifdef DFM_EMU
  for (int g = 0; g < nch; ++g) {
    const int s0 = g * Lc, len = (n - s0 < Lc) ? n - s0 : Lc;
    for (int s = 0; s < len; ++s) {
      int t = t0 + dir * (s0 + s);
      if (g > 0 && s == 0) continue;                        // zero incoming state
      double nz[R];
      for (int i = 0; i < R; ++i) { double a = Z[ZI(t, i)]; for (int j = 0; j < R; ++j) a += Cf[i * R + j] * Z[ZI(t - dir, j)]; nz[i] = a; }
      for (int i = 0; i < R; ++i) Z[ZI(t, i)] = nz[i];
    }
  }
#else
  // state of the group's chunk lives in registers (lane gl = component gl); the matrix-vector product
  // gathers the 8 components with width-8 shuffles: no shared-memory round trip on the serial chain
  const int g = threadIdx.x >> 3, gl = threadIdx.x & 7;           // ng groups >= nch
  const int s0 = g * Lc;
  const int len = (g < nch) ? ((n - s0 < Lc) ? n - s0 : Lc) : 0;
  const bool lane_on = gl < R;
  double cf[R];
#pragma unroll
  for (int j = 0; j < R; ++j) cf[j] = lane_on ? Cf[gl * R + j] : 0.0;
  double cur = (g == 0 && lane_on) ? Z[ZI(t0 - dir, gl)] : 0.0;        // chunk 0 continues the true state, the others start from 0
  {
    double u = (lane_on && len > 0) ? Z[ZI(t0 + dir * s0, gl)] : 0.0;
    for (int s = 0; s < Lc; ++s) {                                     // uniform trip count: every lane takes part in the shuffles
      const bool on = lane_on && s < len;
      const double un = (lane_on && s + 1 < len) ? Z[ZI(t0 + dir * (s0 + s + 1), gl)] : 0.0;   // next input, off the chain
      double a0 = u, a1 = 0.0;
#pragma unroll
      for (int j = 0; j < R; ++j) {
        const double v = __shfl_sync(0xffffffffu, cur, j, 8);
        if (j & 1) a1 += cf[j] * v; else a0 += cf[j] * v;
      }
      const double nx = a0 + a1;
      if (on) { Z[ZI(t0 + dir * (s0 + s), gl)] = nx; cur = nx; }
      u = un;
    }
  }
#endif
  BLK_SYNC();
  if (nch > 1) {
    // ---- boundary propagation: bnd[g] = true state entering chunk g (g >= 1)
#ifdef DFM_EMU
    if (DFM_WARP == 0) {
      for (int gg = 1; gg < nch; ++gg) {
        const int tend = t0 + dir * (gg * Lc - 1);            // last step of chunk gg-1
        for (int i = DFM_LANE; i < R; i += DFM_WSZ) {
          double a = Z[ZI(tend, i)];
          if (gg > 1) for (int j = 0; j < R; ++j) a += pw[i * R + j] * bnd[(gg - 1) * R + j];
          bnd[gg * R + i] = a;
        }
        DFM_WSYNC();
      }
    }
#else
    if (pl1 && nch <= 32) {
      // Kogge-Stone over the chunk-end states: after level l, x_g = sum_{j < 2^(l+1)} pw^j e_{g-j}; the level
      // matrix pw^(2^l) is read row-wise from shared memory, x_{g-2^l} through a double-buffered exchange array
      double x = cur;                                                    // e_g: local end state of my chunk (true for chunk 0)
      double* xb = bnd + (size_t)(ng + 1) * R;                           // [2][ng][R]
      const double* lv[5] = {pw, pl1, pl2, pl3, pl4};
#pragma unroll
      for (int lvl = 0; lvl < 5; ++lvl) {
        const int off = 1 << lvl;
        if (off < nch) {                                                 // uniform
          double* xw = xb + (size_t)(lvl & 1) * ng * R;
          if (lane_on && g < nch) xw[g * R + gl] = x;
          BLK_SYNC();
          const bool use = lane_on && g >= off && g < nch;
          const double yv = use ? xw[(g - off) * R + gl] : 0.0;
          const double* prow = lv[lvl] + gl * R;
          double a0 = x, a1 = 0.0;
#pragma unroll
          for (int j = 0; j < R; ++j) {
            const double v = __shfl_sync(0xffffffffu, yv, j, 8);
            const double pj = lane_on ? prow[j] : 0.0;
            if (j & 1) a1 += pj * v; else a0 += pj * v;
          }
          x = a0 + a1;
        }
      }
      if (lane_on && g + 1 < nch) bnd[(g + 1) * R + gl] = x;             // true end state of chunk g = state entering chunk g+1
    } else if (DFM_WARP == 0) {
      const int gl = threadIdx.x & 7;
      const bool lane_on = gl < R;
      double pr[R];
#pragma unroll
      for (int j = 0; j < R; ++j) pr[j] = lane_on ? pw[gl * R + j] : 0.0;
      double b = lane_on ? Z[ZI(t0 + dir * (Lc - 1), gl)] : 0.0;          // end of chunk 0 = true state entering chunk 1
      double loc = (lane_on && nch > 2) ? Z[ZI(t0 + dir * (2 * Lc - 1), gl)] : 0.0;
      for (int gg = 1; gg < nch; ++gg) {
        if (lane_on && threadIdx.x < 8) bnd[gg * R + gl] = b;
        const double locn = (lane_on && gg + 2 < nch) ? Z[ZI(t0 + dir * ((gg + 2) * Lc - 1), gl)] : 0.0;
        double a0 = loc, a1 = 0.0;
#pragma unroll
        for (int j = 0; j < R; ++j) {
          const double v = __shfl_sync(0xffffffffu, b, j, 8);
          if (j & 1) a1 += pr[j] * v; else a0 += pr[j] * v;
        }
        b = a0 + a1;                                                        // true end state of chunk gg = entering state of chunk gg+1
        loc = locn;
      }
    }
#endif
    BLK_SYNC();
    // ---- pass 2: add Cf^(s+1) bnd[g]
#ifdef DFM_EMU
    for (int g = 1; g < nch; ++g) {
      const int s0 = g * Lc, len = (n - s0 < Lc) ? n - s0 : Lc;
      double c[R], c2[R];
      for (int i = 0; i < R; ++i) c[i] = bnd[g * R + i];
      for (int s = 0; s < len; ++s) {
        int t = t0 + dir * (s0 + s);
        for (int i = 0; i < R; ++i) { double a = 0.0; for (int j = 0; j < R; ++j) a += Cf[i * R + j] * c[j]; c2[i] = a; }
        for (int i = 0; i < R; ++i) { c[i] = c2[i]; Z[ZI(t, i)] += c[i]; }
      }
    }
#else
    {
      const bool act2 = lane_on && g > 0 && len > 0;
      double c = act2 ? bnd[g * R + gl] : 0.0;
      for (int s = 0; s < Lc; ++s) {
        double a0 = 0.0, a1 = 0.0;
#pragma unroll
        for (int j = 0; j < R; ++j) {
          const double v = __shfl_sync(0xffffffffu, c, j, 8);
          if (j & 1) a1 += cf[j] * v; else a0 += cf[j] * v;
        }
        c = a0 + a1;
        if (act2 && s < len) Z[ZI(t0 + dir * (s0 + s), gl)] += c;
      }
    }
#endif
    BLK_SYNC();
  }
#undef BLK_SYNC
}

// ================================================================================================
#ifdef DFM_EMU
#define DFM_FUSED_BOUNDS
#else
#define DFM_FUSED_BOUNDS __launch_bounds__(128, 3)
#endif
template <int R>
__global__ void DFM_FUSED_BOUNDS k_em_fused(FusedArgs a) {
  DFM_SMEM(sm);
  constexpr int RR = R * R, NP = R * (R + 1) / 2;
  const int T = a.T, N = a.N;
  // ---- shared layout
  const int Tp = pad4mod16(T), Np = pad4mod16(N);
  double* Z = sm;                          // [FZ][Tp] component-major
  double* Lam = Z + (size_t)FZ * Tp;       // [R][Np] component-major
  double* rinv = Lam + (size_t)R * Np;     // [N]
  double* Rv = rinv + N;                   // [N]
  double* sxx = Rv + N;                    // [N]
  double* mats = sxx + N;
  double* M = mats;            double* Q = M + RR;        double* C = Q + RR;        double* Pp = C + RR;
  double* Pi = Pp + RR;        double* Pf = Pi + RR;      double* Wm = Pf + RR;      double* G = Wm + RR;
  double* Phi = G + RR;        double* Jm = Phi + RR;     double* Pn = Jm + RR;      double* T1 = Pn + RR;
  double* T2 = T1 + RR;        double* Ps = T2 + RR;      double* Psn = Ps + RR;     double* SPall = Psn + RR;
  double* SP00 = SPall + RR;   double* SPff2 = SP00 + RR; double* SP11 = SPff2 + RR; double* Sm = SP11 + RR;
  double* S11m = Sm + RR;      double* Pfinf = S11m + RR; double* Phinf = Pfinf + RR; double* Jinf = Phinf + RR;
  double* Winf = Jinf + RR;    double* Ppinf = Winf + RR; double* IJM = Ppinf + RR;  double* Pfprev = IJM + RR;
  double* tmp = Pfprev + RR;               // 2R
  double* red = tmp + 2 * R;               // 40
  double* scal = red + 40;                 // 8: [0]=slr [1]=ld_inf [2]=qsum
  int* ctl = (int*)(scal + 8);             // [0]=nE [1]=tb [2]=bad [3]=frozen
  double* bnd = scal + 16;                 // [0,17R) chunk-boundary states, [17R,49R) per-group ping-pong vectors, [64R, 64R+RR) scratch
  double* scr = a.scratch + (size_t)DFM_BX * T * FUSED_SCR(R);
  // per explicit step t: scr[t*SCR + {0:Pf, RR:Phi, 2RR:J, 3RR:W, 4RR:Ps, 5RR: ld}]
  const double eps = 1e-14;

  for (int b = DFM_BX; b < a.B; b += DFM_GX) {
    const double* X = a.X + (size_t)b * T * N;
    // ---- load parameters (global column-major -> shared row-major)
    for (int e = DFM_TID; e < N * R; e += DFM_NT) { int i = e % N, c = e / N; Lam[LI(i, c)] = a.Lam[(size_t)b * N * R + e]; }
    for (int e = DFM_TID; e < N; e += DFM_NT) Rv[e] = a.R[(size_t)b * N + e];
    for (int e = DFM_TID; e < RR; e += DFM_NT) {
      int i = e / R, j = e % R;
      M[e] = a.A[(size_t)b * RR + i + R * j]; Q[e] = a.Q[(size_t)b * RR + i + R * j];
    }
    if (DFM_TID == 0) ctl[2] = 0;
    DFM_SYNC();
    int it = 0, status = 0;
    double ll_prev = 0.0;
    for (; it < a.max_iter; ++it) {
      // ---------------------------------------------------------------- P0: prep
      double slr_p = 0.0;
      for (int i = DFM_TID; i < N; i += DFM_NT) { double rv = Rv[i]; rinv[i] = 1.0 / rv; slr_p += log(rv); if (!(rv > 0.0)) ctl[2] = 1; }
      slr_p = block_sum(slr_p, red);
      if (DFM_TID == 0) scal[0] = slr_p;
      for (int e = DFM_TID; e < RR; e += DFM_NT) {
        int i = e / R, j = e % R;
        double s = 0.0;
        for (int n = 0; n < N; ++n) s += Lam[LI(n, i)] * rinv[n] * Lam[LI(n, j)];
        C[e] = s;
      }
      DFM_SYNC();
      // ---------------------------------------------------------------- P1: E-step contraction (panel pass 1)
      double qacc = 0.0;
#ifdef DFM_EMU
      for (int t = 0; t < T; ++t) {
        for (int c = 0; c < FZ; ++c) Z[ZI(t, c)] = 0.0;
        for (int n = 0; n < N; ++n) {
          double x = X[(size_t)n * T + t], xr = x * rinv[n];
          qacc += x * xr;
          for (int c = 0; c < R; ++c) Z[ZI(t, c)] += xr * Lam[LI(n, c)];
        }
      }
#else
      {
        // flattened (row-block, 40-series batch) loop, software pipelined: the loads of batch q+1 are
        // in flight while the 10 DMMAs of batch q issue (two register buffers of 10 doubles)
        const int lane = DFM_LANE, lr = lane >> 2, lc = lane & 3;
        const int nrb = (T + 7) / 8, nbt = (N + 39) / 40;
        const int my_rb = (nrb - DFM_WARP + DFM_NWARP - 1) / DFM_NWARP;      // row blocks of this warp
        const int nq = my_rb * nbt;
        double bufA[10], bufB[10];
        double d0 = 0.0, d1 = 0.0;
#define DFM_E_LOAD(buf, q_)                                                                         \
        { const int rb_ = DFM_WARP + DFM_NWARP * ((q_) / nbt), i0_ = ((q_) % nbt) * 40;             \
          const int t_ = rb_ * 8 + lr; const bool tok_ = t_ < T; const double* xp_ = X + (tok_ ? t_ : 0); \
          _Pragma("unroll") for (int u = 0; u < 10; ++u) { const int n_ = i0_ + 4 * u + lc;          \
            buf[u] = (tok_ && n_ < N) ? __ldg(xp_ + (size_t)n_ * T) : 0.0; } }
#define DFM_E_USE(buf, q_)                                                                          \
        { const int rb_ = DFM_WARP + DFM_NWARP * ((q_) / nbt), bt_ = (q_) % nbt, i0_ = bt_ * 40;     \
          _Pragma("unroll") for (int u = 0; u < 10; ++u) { const int n_ = i0_ + 4 * u + lc;          \
            if (i0_ + 4 * u < N) {                                                                   \
              const double ri_ = (n_ < N) ? rinv[n_] : 0.0; const double ar_ = buf[u] * ri_;         \
              qacc += buf[u] * ar_;                                                                  \
              const double bv_ = (n_ < N && lr < R) ? Lam[LI(n_, lr)] : 0.0;                        \
              asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n" \
                           : "+d"(d0), "+d"(d1) : "d"(ar_), "d"(bv_)); } }                           \
          if (bt_ == nbt - 1) { const int t_ = rb_ * 8 + lr;                                         \
            if (t_ < T) { Z[ZI(t_, 2 * lc)] = d0; Z[ZI(t_, 2 * lc + 1)] = d1; }                  \
            d0 = 0.0; d1 = 0.0; } }
        if (nq > 0) DFM_E_LOAD(bufA, 0);
        for (int q = 0; q < nq; q += 2) {
          if (q + 1 < nq) DFM_E_LOAD(bufB, q + 1);
          DFM_E_USE(bufA, q);
          if (q + 2 < nq) DFM_E_LOAD(bufA, q + 2);
          if (q + 1 < nq) DFM_E_USE(bufB, q + 1);
        }
#undef DFM_E_LOAD
#undef DFM_E_USE
      }
#endif
      qacc = block_sum(qacc, red);
      if (DFM_TID == 0) scal[2] = qacc;
      DFM_SYNC();
      // ---------------------------------------------------------------- P2: covariance chain (warp 0, data independent)
      if (DFM_WARP == 0) {
        int* bad = &ctl[2];
        // forward
        for (int e = DFM_LANE; e < RR; e += DFM_WSZ) { int i = e / R, j = e % R; Pp[e] = a.P0[(size_t)b * RR + i + R * j]; }
        DFM_WSYNC();
        int nE = T, frozen_at = -1, t = 0;
        while (t < T) {
          double ldp = w_inv<R>(Pi, Pp, tmp, bad);
          for (int e = DFM_LANE; e < RR; e += DFM_WSZ) Wm[e] = Pi[e] + C[e];
          DFM_WSYNC();
          double ldw = w_inv<R>(Pf, Wm, tmp, bad);
          w_gemm<R>(G, Pf, false, Pi, false);
          w_gemm<R>(Phi, G, false, M, false);
          if (t >= 1) { w_gemm<R>(T1, Pfprev, false, M, true); w_gemm<R>(Jm, T1, false, Pi, false); }   // J_{t-1}
          w_gemm<R>(T1, M, false, Pf, false);
          w_gemm<R>(Pn, T1, false, M, true);
          for (int e = DFM_LANE; e < RR; e += DFM_WSZ) Pn[e] += Q[e];
          DFM_WSYNC();
          w_sym<R>(Pn);
          double* s_ = scr + (size_t)t * FUSED_SCR(R);
          double dmax = 0.0, pmax = 0.0;
          for (int e = DFM_LANE; e < RR; e += DFM_WSZ) {
            s_[e] = Pf[e]; s_[RR + e] = Phi[e]; s_[3 * RR + e] = Wm[e];
            if (t >= 1) (s_ - FUSED_SCR(R))[2 * RR + e] = Jm[e];
            dmax = fmax(dmax, fabs(Pn[e] - Pp[e])); pmax = fmax(pmax, fabs(Pp[e]));
            Pfprev[e] = Pf[e];
          }
          if (DFM_LANE == 0) s_[5 * RR] = ldp + ldw;
          dmax = w_max(dmax); pmax = w_max(pmax);
          DFM_WSYNC();
          if (frozen_at >= 0 && t == frozen_at + 1) {
            nE = t + 1;
            for (int e = DFM_LANE; e < RR; e += DFM_WSZ) { Pfinf[e] = Pf[e]; Phinf[e] = Phi[e]; Winf[e] = Wm[e]; }
            if (DFM_LANE == 0) scal[1] = ldp + ldw;
            DFM_WSYNC();
            w_gemm<R>(T1, Pf, false, M, true);
            w_gemm<R>(Jinf, T1, false, Pi, false);                 // J_inf = Pf_inf M' Pi_inf
            break;
          }
          if (frozen_at < 0 && dmax <= eps * pmax) frozen_at = t;
          for (int e = DFM_LANE; e < RR; e += DFM_WSZ) Pp[e] = Pn[e];
          DFM_WSYNC();
          ++t;
        }
        const int frozen = nE < T;
        // backward covariance chain + covariance parts of the moment sums
        for (int e = DFM_LANE; e < RR; e += DFM_WSZ) {
          double v = frozen ? Pfinf[e] : (scr + (size_t)(T - 1) * FUSED_SCR(R))[e];
          Psn[e] = v; SPall[e] = v; SPff2[e] = v; SP00[e] = 0.0; SP11[e] = 0.0;
          (scr + (size_t)(T - 1) * FUSED_SCR(R))[4 * RR + e] = v;
        }
        DFM_WSYNC();
        const int lo = frozen ? nE - 1 : T;
        int tb = -1;                        // frozen smoothed range is [lo, tb)
        t = T - 2;
        while (t >= 0) {
          const double* pf_t = (t < nE) ? scr + (size_t)t * FUSED_SCR(R) : Pfinf;
          const double* j_t = (t < nE - 1) ? scr + (size_t)t * FUSED_SCR(R) + 2 * RR : Jinf;
          // Pp_{t+1} = M Pf_t M' + Q (recomputed: cheaper than storing)
          w_gemm<R>(T1, M, false, pf_t, false);
          w_gemm<R>(T2, T1, false, M, true);
          for (int e = DFM_LANE; e < RR; e += DFM_WSZ) T2[e] = Psn[e] - (T2[e] + Q[e]);
          DFM_WSYNC();
          w_sym<R>(T2);                                           // D = Ps_{t+1} - Pp_{t+1}
          w_gemm<R>(T1, j_t, false, T2, false);
          w_gemm<R>(Ps, T1, false, j_t, true);
          for (int e = DFM_LANE; e < RR; e += DFM_WSZ) Ps[e] += pf_t[e];
          DFM_WSYNC();
          w_sym<R>(Ps);
          w_gemm<R>(T1, Psn, false, j_t, true);                    // Ps_{t+1} J_t'
          double dmax = 0.0, pmax = 0.0;
          for (int e = DFM_LANE; e < RR; e += DFM_WSZ) {
            SP11[e] += T1[e]; SPall[e] += Ps[e]; SP00[e] += Ps[e];
            if (t >= 1) SPff2[e] += Ps[e];
            (scr + (size_t)t * FUSED_SCR(R))[4 * RR + e] = Ps[e];
            dmax = fmax(dmax, fabs(Ps[e] - Psn[e])); pmax = fmax(pmax, fabs(Ps[e]));
          }
          dmax = w_max(dmax); pmax = w_max(pmax);
          DFM_WSYNC();
          bool conv = frozen && t > lo && dmax <= eps * pmax;
          for (int e = DFM_LANE; e < RR; e += DFM_WSZ) Psn[e] = Ps[e];
          DFM_WSYNC();
          if (conv) {
            tb = t;
            double cnt = (double)(t - lo);
            w_gemm<R>(T1, Ps, false, Jinf, true);
            for (int e = DFM_LANE; e < RR; e += DFM_WSZ) {
              SPall[e] += cnt * Ps[e]; SP00[e] += cnt * Ps[e];
              SPff2[e] += ((lo >= 1) ? cnt : cnt - 1.0) * Ps[e];
              SP11[e] += cnt * T1[e];
              Ppinf[e] = Ps[e];                                  // Ps_inf (smoothed covariance of the frozen range)
            }
            DFM_WSYNC();
            t = lo - 1;
          } else --t;
        }
        if (DFM_LANE == 0) { ctl[0] = nE; ctl[1] = tb; ctl[3] = frozen; }
        // I - J_inf M  (for the parallel pre-pass of the backward mean recursion)
        if (frozen) {
          w_gemm<R>(IJM, Jinf, false, M, false);
          for (int e = DFM_LANE; e < RR; e += DFM_WSZ) { int i = e / R, j = e % R; IJM[e] = ((i == j) ? 1.0 : 0.0) - IJM[e]; }
        }
        DFM_WSYNC();
      }
      DFM_SYNC();
      const int nE = ctl[0], frozen = ctl[3];
      // ---------------------------------------------------------------- P3: forward means
      // parallel pre-pass over the frozen range: Z[t] <- Pf_inf b_t
      for (int t = nE + DFM_TID; t < T; t += DFM_NT) {
        double bb[R], u[R];
#pragma unroll
        for (int j = 0; j < R; ++j) bb[j] = Z[ZI(t, j)];
#pragma unroll
        for (int i = 0; i < R; ++i) { double s = 0.0;
#pragma unroll
          for (int j = 0; j < R; ++j) s += Pfinf[i * R + j] * bb[j]; u[i] = s; }
#pragma unroll
        for (int i = 0; i < R; ++i) Z[ZI(t, i)] = u[i];
      }
      DFM_SYNC();
      if (DFM_WARP == 0) {
        // explicit steps
        for (int t = 0; t < nE; ++t) {
          const double* s_ = scr + (size_t)t * FUSED_SCR(R);
          for (int i = DFM_LANE; i < R; i += DFM_WSZ) {
            double s = 0.0;
            for (int j = 0; j < R; ++j) s += s_[i * R + j] * Z[ZI(t, j)];                 // Pf_t b_t
            if (t >= 1) for (int j = 0; j < R; ++j) s += s_[RR + i * R + j] * Z[ZI(t - 1, j)];   // Phi_t zf_{t-1}
            tmp[i] = s;
          }
          DFM_WSYNC();
          for (int i = DFM_LANE; i < R; i += DFM_WSZ) Z[ZI(t, i)] = tmp[i];
          DFM_WSYNC();
        }
      }
      DFM_SYNC();
      // frozen steps: z_t = Phi_inf z_{t-1} + u_t, parallel in time over the CTA
      if (frozen) blk_recur<R>(Z, Tp, Phinf, T1, T2, bnd, (nE > 0 ? nE : 1), T - (nE > 0 ? nE : 1), +1, 128);
      // ---------------------------------------------------------------- P4: log-likelihood (parallel over t)
      double llp = 0.0;
      for (int t = DFM_TID; t < T; t += DFM_NT) {
        const double* Wt = (t < nE) ? scr + (size_t)t * FUSED_SCR(R) + 3 * RR : Winf;
        double ldt = (t < nE) ? (scr + (size_t)t * FUSED_SCR(R))[5 * RR] : scal[1];
        double zp[R], d[R];
#pragma unroll
        for (int i = 0; i < R; ++i) { double s = 0.0; if (t >= 1) {
#pragma unroll
            for (int j = 0; j < R; ++j) s += M[i * R + j] * Z[ZI(t - 1, j)]; }
          zp[i] = s; d[i] = Z[ZI(t, i)] - s; }
        double quad = 0.0;
#pragma unroll
        for (int i = 0; i < R; ++i) {
          double cz = 0.0, g = 0.0;
#pragma unroll
          for (int j = 0; j < R; ++j) { cz += C[i * R + j] * zp[j]; g += Wt[i * R + j] * d[j]; }
          quad -= zp[i] * cz + 2.0 * zp[i] * g + g * d[i];
        }
        llp += -0.5 * ((double)N * 1.8378770664093454835606594728112 + scal[0] + ldt + quad);
      }
      llp = block_sum(llp, red);
      const double ll = llp - 0.5 * scal[2];
      // ---------------------------------------------------------------- P5: backward means
      if (frozen) {
        int lo = nE - 1;
        for (int t = lo + DFM_TID; t < T - 1; t += DFM_NT) {       // Z[t] <- (I - J_inf M) zf_t
          double zz[R], v[R];
#pragma unroll
          for (int j = 0; j < R; ++j) zz[j] = Z[ZI(t, j)];
#pragma unroll
          for (int i = 0; i < R; ++i) { double s = 0.0;
#pragma unroll
            for (int j = 0; j < R; ++j) s += IJM[i * R + j] * zz[j]; v[i] = s; }
#pragma unroll
          for (int i = 0; i < R; ++i) Z[ZI(t, i)] = v[i];
        }
      }
      DFM_SYNC();
      // frozen range: z_t = J_inf z_{t+1} + v_t, parallel in time over the CTA
      if (frozen) blk_recur<R>(Z, Tp, Jinf, T1, T2, bnd, T - 2, (T - 2) - (nE - 1) + 1, -1, 128);
      if (DFM_WARP == 0) {
        const int lo = frozen ? nE - 1 : T;
        // explicit range: zs_t = zf_t + J_t (zs_{t+1} - M zf_t)
        for (int t = (lo - 1 < T - 2 ? lo - 1 : T - 2); t >= 0; --t) {
          const double* j_t = scr + (size_t)t * FUSED_SCR(R) + 2 * RR;
          for (int i = DFM_LANE; i < R; i += DFM_WSZ) { double s = Z[ZI(t + 1, i)]; for (int j = 0; j < R; ++j) s -= M[i * R + j] * Z[ZI(t, j)]; tmp[i] = s; }
          DFM_WSYNC();
          for (int i = DFM_LANE; i < R; i += DFM_WSZ) { double s = Z[ZI(t, i)]; for (int j = 0; j < R; ++j) s += j_t[i * R + j] * tmp[j]; tmp[R + i] = s; }
          DFM_WSYNC();
          for (int i = DFM_LANE; i < R; i += DFM_WSZ) Z[ZI(t, i)] = tmp[R + i];
          DFM_WSYNC();
        }
      }
      DFM_SYNC();
      // ---------------------------------------------------------------- P7: mean parts of the moment sums
      for (int e = DFM_TID; e < 2 * RR; e += DFM_NT) {
        int which = e / RR, ee = e % RR, i = ee / R, j = ee % R;
        double s = 0.0;
        if (which == 0) { for (int t = 0; t < T; ++t) s += Z[ZI(t, i)] * Z[ZI(t, j)]; Sm[ee] = s; }
        else { for (int t = 1; t < T; ++t) s += Z[ZI(t, i)] * Z[ZI(t - 1, j)]; S11m[ee] = s; }
      }
      DFM_SYNC();
      // ---------------------------------------------------------------- P8: M-step contraction (panel pass 2)
#ifdef DFM_EMU
      for (int n = 0; n < N; ++n) {
        double s2 = 0.0, acc[R];
        for (int c = 0; c < R; ++c) acc[c] = 0.0;
        for (int t = 0; t < T; ++t) { double x = X[(size_t)n * T + t]; s2 += x * x; for (int c = 0; c < R; ++c) acc[c] += x * Z[ZI(t, c)]; }
        for (int c = 0; c < R; ++c) Lam[LI(n, c)] = acc[c];
        sxx[n] = s2;
      }
#else
      {
        const int lane = DFM_LANE, lr = lane >> 2, lc = lane & 3;
        const int nsb = (N + 7) / 8, nbt = (T + 39) / 40;
        const int my_sb = (nsb - DFM_WARP + DFM_NWARP - 1) / DFM_NWARP;
        const int nq = my_sb * nbt;
        double bufA[10], bufB[10];
        double d0 = 0.0, d1 = 0.0, s2 = 0.0;
#define DFM_M_LOAD(buf, q_)                                                                         \
        { const int sb_ = DFM_WARP + DFM_NWARP * ((q_) / nbt), t0_ = ((q_) % nbt) * 40;              \
          const int n_ = sb_ * 8 + lr; const bool nok_ = n_ < N; const double* xp_ = X + (size_t)(nok_ ? n_ : 0) * T; \
          _Pragma("unroll") for (int u = 0; u < 10; ++u) { const int t_ = t0_ + 4 * u + lc;          \
            buf[u] = (nok_ && t_ < T) ? __ldg(xp_ + t_) : 0.0; } }
#define DFM_M_USE(buf, q_)                                                                          \
        { const int sb_ = DFM_WARP + DFM_NWARP * ((q_) / nbt), bt_ = (q_) % nbt, t0_ = bt_ * 40;     \
          _Pragma("unroll") for (int u = 0; u < 10; ++u) { const int t_ = t0_ + 4 * u + lc;          \
            if (t0_ + 4 * u < T) {                                                                   \
              s2 += buf[u] * buf[u];                                                                 \
              const double bv_ = (t_ < T) ? Z[ZI(t_, lr)] : 0.0;                                   \
              asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n" \
                           : "+d"(d0), "+d"(d1) : "d"(buf[u]), "d"(bv_)); } }                        \
          if (bt_ == nbt - 1) { const int n_ = sb_ * 8 + lr;                                         \
            s2 += __shfl_xor_sync(0xffffffffu, s2, 1); s2 += __shfl_xor_sync(0xffffffffu, s2, 2);    \
            if (n_ < N) { if (2 * lc < R) Lam[LI(n_, 2 * lc)] = d0; if (2 * lc + 1 < R) Lam[LI(n_, 2 * lc + 1)] = d1; \
                          if (lc == 0) sxx[n_] = s2; }                                               \
            d0 = 0.0; d1 = 0.0; s2 = 0.0; } }
        if (nq > 0) DFM_M_LOAD(bufA, 0);
        for (int q = 0; q < nq; q += 2) {
          if (q + 1 < nq) DFM_M_LOAD(bufB, q + 1);
          DFM_M_USE(bufA, q);
          if (q + 2 < nq) DFM_M_LOAD(bufA, q + 2);
          if (q + 1 < nq) DFM_M_USE(bufB, q + 1);
        }
#undef DFM_M_LOAD
#undef DFM_M_USE
      }
#endif
      DFM_SYNC();
      // ---------------------------------------------------------------- P9: M-step solves
      if (DFM_WARP == 0) {
        int* bad = &ctl[2];
        // measurement: S = SffAll;  Lam_i = S^-1 Sxf_i
        for (int e = DFM_LANE; e < RR; e += DFM_WSZ) T1[e] = Sm[e] + SPall[e];
        DFM_WSYNC();
        w_sym<R>(T1);
        w_inv<R>(G, T1, tmp, bad);                                 // G = S^-1, T1 = S
        // transition: A = S11 S00^-1 ; Q = (Sff2 - A S11') / (T-1)
        for (int e = DFM_LANE; e < RR; e += DFM_WSZ) {
          int i = e / R, j = e % R;
          Pp[e] = Sm[e] - Z[ZI(T - 1, i)] * Z[ZI(T - 1, j)] + SP00[e];        // S00
          Pi[e] = Sm[e] - Z[ZI(0, i)] * Z[ZI(0, j)] + SPff2[e];                    // Sff2
          Pf[e] = S11m[e] + SP11[e];                                                    // S11
        }
        DFM_WSYNC();
        w_sym<R>(Pp);
        w_inv<R>(Wm, Pp, tmp, bad);
        w_gemm<R>(Phi, Pf, false, Wm, false);                      // A_new
        w_gemm<R>(Pn, Phi, false, Pf, true);                       // A S11'
        for (int e = DFM_LANE; e < RR; e += DFM_WSZ) Pn[e] = (Pi[e] - Pn[e]) / (double)(T - 1);
        DFM_WSYNC();
        w_sym<R>(Pn);                                              // Q_new
      }
      DFM_SYNC();
      for (int n = DFM_TID; n < N; n += DFM_NT) {
        double sx[R], lam[R];
#pragma unroll
        for (int c = 0; c < R; ++c) sx[c] = Lam[LI(n, c)];
        double q1 = 0.0, q2 = 0.0;
#pragma unroll
        for (int i = 0; i < R; ++i) { double s = 0.0;
#pragma unroll
          for (int j = 0; j < R; ++j) s += G[i * R + j] * sx[j]; lam[i] = s; q1 += s * sx[i]; }
#pragma unroll
        for (int i = 0; i < R; ++i) { double s = 0.0;
#pragma unroll
          for (int j = 0; j < R; ++j) s += T1[i * R + j] * lam[j]; q2 += lam[i] * s; }
#pragma unroll
        for (int c = 0; c < R; ++c) Lam[LI(n, c)] = lam[c];
        Rv[n] = (sxx[n] - 2.0 * q1 + q2) / (double)T;
      }
      DFM_SYNC();
      for (int e = DFM_TID; e < RR; e += DFM_NT) { M[e] = Phi[e]; Q[e] = Pn[e]; }
      if (DFM_TID == 0) a.loglik[(size_t)b * a.max_iter + it] = ll;
      DFM_SYNC();
      if (ctl[2] || !(ll == ll)) { status = 3; ++it; break; }
      bool conv = (it >= 1) && fabs(ll - ll_prev) <= a.tol * 0.5 * (fabs(ll) + fabs(ll_prev));
      ll_prev = ll;
      if (conv) { ++it; break; }
    }
    // ---- outputs
    for (int e = DFM_TID; e < N * R; e += DFM_NT) { int i = e % N, c = e / N; a.Lam[(size_t)b * N * R + e] = Lam[LI(i, c)]; }
    for (int e = DFM_TID; e < N; e += DFM_NT) a.R[(size_t)b * N + e] = Rv[e];
    for (int e = DFM_TID; e < RR; e += DFM_NT) {
      int i = e % R, j = e / R;                                   // column-major out
      a.A[(size_t)b * RR + e] = M[i * R + j]; a.Q[(size_t)b * RR + e] = Q[i * R + j];
    }
    for (int e = DFM_TID; e < T * R; e += DFM_NT) { int t = e % T, c = e / T; a.Fs[(size_t)b * T * R + e] = Z[ZI(t, c)]; }
    {
      const int nE = ctl[0], tb = ctl[1], frozen = ctl[3];
      const int lo = frozen ? nE - 1 : T;
      for (int e = DFM_TID; e < T * NP; e += DFM_NT) {
        int t = e % T, pe = e / T;
        int i = 0; while ((i + 1) * (i + 2) / 2 <= pe) ++i;
        int j = pe - i * (i + 1) / 2;
        bool in_frozen = frozen && tb >= 0 && t >= lo && t < tb;
        double v = in_frozen ? Ppinf[i * R + j] : (scr + (size_t)t * FUSED_SCR(R))[4 * RR + i * R + j];
        a.PsF[(size_t)b * T * NP + e] = v;
      }
    }
    if (DFM_TID == 0) { a.iters[b] = it > a.max_iter ? a.max_iter : it; a.status[b] = status; }
    DFM_SYNC();
  }
}

template <int R>
inline size_t fused_smem_doubles(int T, int N) {
  return (size_t)FZ * pad4mod16(T) + (size_t)R * pad4mod16(N) + 3 * (size_t)N + 30 * (size_t)R * R + 2 * R + 40 + 8 + 8 + 64 * R + (size_t)R * R + 8;
}

}  // namespace dfm
