// dfm_kernels_fused2.cuh -- TMA-fed fused per-panel EM kernel k_em_fused2<R> (the default for balanced panels with
// p = 1, r <= 8, even T) and the fused ALS sweep kernel k_als_fused2<R>.  See DESIGN.md section 4.1.
//  * 256 threads in three roles: warp 0 = TMA producer during the two panel passes, warps 1..6 = DMMA consumers,
//    warp 7 = "chain warp" (covariance recursions, moment sums, r x r M-step solves -- all data independent or
//    r x r sized, overlapped with the passes and with the mean recursions);
//  * both passes stream the column-major panel through ONE 2-D tensor-map copy per stage (cp.async.bulk.tensor.2d,
//    SASS UTMALDG; box = F2_TC periods x 8 series) into an F2_S-stage shared-memory ring guarded by full/empty
//    mbarriers (tools/bench_stream.cu and tools/bench_tma2d.cu compare the load schemes at this occupancy);
//  * E pass: each consumer warp keeps the 8x8 accumulators of its row blocks in registers across all series blocks;
//    M pass: S_xf partial tiles per consumer warp + deterministic cross-warp reduction per series block;
//  * the ring is idle between the passes and doubles as storage for the explicit covariance steps and the level
//    matrices of the backward scan (no dependent global-memory round trips on the serial path);
//  * streaming host path: the kernel may be launched before its panels are on the device (FusedArgs::ready/done).
// Requires T even (16-byte aligned column runs); otherwise dfm_em_kalman uses k_em_fused.
#pragma once
#include <algorithm>
#include "dfm_kernels_fused.cuh"
#ifdef DFM_EMU
struct CUtensorMap { char opaque[128]; };
#define DFM_GRID_CONSTANT
#else
#include <cuda.h>          // CUtensorMap (types only; the encoder is fetched with cudaGetDriverEntryPoint)
#define DFM_GRID_CONSTANT __grid_constant__
#endif

namespace dfm {

#ifndef F2_SBS
#define F2_SBS 1        // 8-series blocks per stage (= per tensor-map copy): a copy has a fixed cost whatever its size
#endif                  // (tools/bench_tma2d.cu), so wider stages raise the rate a single CTA can stream at
#ifndef F2_S
#define F2_S (3 / F2_SBS)   // ring stages (the ring keeps its size: F2_S * F2_SBS * 8 * F2_TS doubles)
#endif
#define F2_STG (F2_SBS * 8 * F2_TS)   // doubles per stage
#ifndef F2_TC
#define F2_TC 172       // periods per stage == row pitch in the ring; must be == 4 or 12 (mod 16) so that the
#endif                  // DMMA fragment loads are bank-conflict free, and <= 256 (TMA box limit).  A copy costs about
                        // the same whatever its size, so T = 500 in 3 chunks of 172 (3 stages) beat 4 of 132 (4 stages)
                        // on c5 by 4 % (H100 SXM 80GB, 700 W, 1980 MHz); 4 chunks of 164 were 7 % slower
#define F2_TS F2_TC     // (box width == chunk stride: no re-read of periods)
#define F2_NCW 6        // consumer warps (warps 1..6; warp 0 = producer, warp 7 = chain / solves)
#define F2_GPARTS_S 4                                    // scalar Gram path: time slices per matrix entry
#define F2_GPARTS ((R == 8) ? (F2_NCW + 1) : F2_GPARTS_S)   // partial Gram matrices (tensor path: one per warp of P3-P5)
#define F2_NRB (((F2_TC + 7) / 8 + F2_NCW - 1) / F2_NCW)   // 8-period DMMA row blocks per consumer warp and stage (E pass)
#define F2_NKC (((F2_TC + 3) / 4 + F2_NCW - 1) / F2_NCW)   // 4-period DMMA k-chunks per consumer warp and stage (M pass)
static_assert(F2_TC % 16 == 4 || F2_TC % 16 == 12, "ring pitch must be 4 or 12 mod 16");
static_assert(F2_TC <= 256 && (F2_TC * 64) % 128 == 0, "TMA box / stage alignment");
#define F2_NEXS(R_) ((F2_S * F2_STG - 4 * (R_) * (R_)) / FUSED_SCR(R_))   // the last 4 R^2 doubles of the idle ring hold scan matrices
#define F2_RTAIL(R_) (F2_S * F2_STG - 4 * (R_) * (R_))
#ifndef F2_L2WIN_PCT
#define F2_L2WIN_PCT 67    // share of L2 for the turn windows of the resident panels (f2_produce; DESIGN.md section 7)
#endif

#ifndef DFM_EMU
__device__ __forceinline__ uint32_t f2_smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void f2_mbar_init(uint64_t* bar, int cnt) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(f2_smem_u32(bar)), "r"(cnt)); }
__device__ __forceinline__ void f2_mbar_expect(uint64_t* bar, uint32_t bytes) { asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(f2_smem_u32(bar)), "r"(bytes) : "memory"); }
__device__ __forceinline__ void f2_mbar_arrive(uint64_t* bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(f2_smem_u32(bar)) : "memory"); }
__device__ __forceinline__ void f2_mbar_wait(uint64_t* bar, uint32_t phase) {
  asm volatile("{\n.reg .pred p;\nWAIT_%=:\nmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n@p bra DONE_%=;\nbra WAIT_%=;\nDONE_%=:\n}" ::"r"(f2_smem_u32(bar)), "r"(phase) : "memory");
}
// one 2-D tensor-map copy (SASS UTMALDG): box F2_TS periods x 8 series of the [T, B*N] view of the batch, with an L2
// eviction policy made by createpolicy
__device__ __forceinline__ void f2_tma_2d(void* dst, const CUtensorMap* tmap, int x, int y, uint64_t* bar, uint64_t policy) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%2, %3}], [%4], %5;"
               ::"r"(f2_smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(x), "r"(y), "r"(f2_smem_u32(bar)), "l"(policy) : "memory");
}

// L2 turn plan.  Each EM iteration (ALS sweep) reads the whole panel twice, but the resident panels are several times
// larger than L2, so a plain stream evicts every line long before its CTA reads it again.  The passes are therefore
// ordered so that each one starts where the previous one ended: the E pass ends on the last period chunk of the high
// series-block groups, and the M pass, which runs backwards over the groups, starts there; the M pass ends on the first
// chunk of the low groups, where the E pass starts.  The last `win` copies of a pass that the next pass re-reads first
// (the turn window) are loaded evict-normal, so that they outlive the evict-first stream until that re-read, a few
// microseconds and one serial phase later; the re-read and every other copy load evict-first (f2_produce).  The host
// splits F2_L2WIN_PCT of L2 over the CTAs of one round of panels (l2_turn_plan): win[0] for the full rounds, win[1] for
// the tail round, whose fewer CTAs may each hold more.
__device__ __forceinline__ int f2_round_win(const int* win, int B, int b) {
  const int G = (int)gridDim.x;
  return (b / G < B / G) ? win[0] : win[1];
}
#endif


#ifndef DFM_EMU
// Position in the ring (every thread keeps its own copy; all copies advance in lock step).
struct F2Ring {
  double* ring; uint64_t* full; uint64_t* empty;
  int rs; uint32_t rph; bool wrap;
  __device__ __forceinline__ void advance() { if (++rs == F2_S) { rs = 0; rph ^= 1; wrap = true; } }
  __device__ __forceinline__ void skip(long long n) { for (long long q = 0; q < n; ++q) advance(); }
};

// Producer side of one pass (warp 0).  Items (c, sb): c_outer selects the loop order.  ONE request per
// stage: a 2-D tensor-map copy of the box [F2_TS periods x 8 series] at (c*F2_TC, row0 + sb*8) of the
// [T, B*N] view of the batch (column runs of 800 B; the box is 4 periods wider than the chunk so that the
// dense row pitch in shared memory is == 4 mod 16, i.e. conflict-free; rows/periods beyond the tensor are
// zero-filled, rows of the next panel are masked by the consumers).  Eight 1-D bulk copies per stage were
// issue-bound (requests serialised over the lanes of a warp: tools/bench_stream.cu).  The E pass (c_outer) runs over the
// series-block groups in ascending order, the M pass in descending order, so that each pass starts on the copies the
// previous one read last.  The turn window (L2 turn plan above; *win is in shared memory) is the last *win groups of
// the last chunk (E pass) or of the first chunk (M pass): it loads evict-normal, the rest evict-first.  Both policies
// are made once per pass: per copy they would lengthen the producer's issue path, which bounds a lone CTA.
__device__ __forceinline__ void f2_produce(F2Ring& rg, const CUtensorMap* tmap, int row0, int T, int N, bool c_outer, const int* win) {
  const int lane = threadIdx.x & 31;
  const int nsb = (N + 8 * F2_SBS - 1) / (8 * F2_SBS), nck = (T + F2_TC - 1) / F2_TC;      // (stages per pass: series-block groups x chunks)
  const int n_out = c_outer ? nck : nsb, n_in = c_outer ? nsb : nck, nw = *win;
  const int wc = c_outer ? nck - 1 : 0, w0 = c_outer ? nsb - nw : 0, w1 = c_outer ? nsb : nw;   // turn window: chunk wc, groups [w0, w1)
  uint64_t pol_win, pol_first;
  asm volatile("createpolicy.fractional.L2::evict_normal.b64 %0, 1.0;" : "=l"(pol_win));
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol_first));
  for (int o = 0; o < n_out; ++o)
    for (int i = 0; i < n_in; ++i) {
      const int c = c_outer ? o : i, sb = c_outer ? i : nsb - 1 - o;
      if (rg.wrap) f2_mbar_wait(&rg.empty[rg.rs], rg.rph ^ 1);
      if (lane == 0) {
        f2_mbar_expect(&rg.full[rg.rs], (uint32_t)(F2_STG * 8));
        f2_tma_2d(rg.ring + (size_t)rg.rs * F2_STG, tmap, c * F2_TC, row0 + sb * 8 * F2_SBS, &rg.full[rg.rs],
                  (c == wc && sb >= w0 && sb < w1) ? pol_win : pol_first);
      }
      __syncwarp();
      rg.advance();
    }
}

// E pass, consumer warp cw (0..F2_NCW-1):  Z[t][:] = sum_n x[t,n] W[n][:]  (W = R^-1 Lam, pre-scaled in P0, or Lam):
// the tile value is the A fragment as it stands, so the load -> DMMA chains carry no scalar work.  SQ: also returns
// this thread's share of sum x^2 (the first ALS sweep).  Period-chunk outer / series-block inner; each warp keeps the
// 8x8 DMMA accumulators of its two row blocks in registers across all series blocks.
template <int R, bool SQ>
__device__ __forceinline__ double f2_consume_E(F2Ring& rg, int cw, int T, int N, int Tp, int Np, double* Z, const double* W) {
  const int lane = threadIdx.x & 31, lr = lane >> 2, lc = lane & 3;
  const int nsg = (N + 8 * F2_SBS - 1) / (8 * F2_SBS), nck = (T + F2_TC - 1) / F2_TC;
  double qacc = 0.0;
  for (int c = 0; c < nck; ++c) {
    const int len = (T - c * F2_TC < F2_TC) ? T - c * F2_TC : F2_TC;
    // row blocks cw, cw + NCW, ...: one independent accumulator pair per (row block, k half) so that no
    // two DMMAs of a series block depend on each other (the chains only link consecutive series blocks)
    double d[F2_NRB][2][2];
#pragma unroll
    for (int j = 0; j < F2_NRB; ++j) { d[j][0][0] = 0.0; d[j][0][1] = 0.0; d[j][1][0] = 0.0; d[j][1][1] = 0.0; }
    for (int sg = 0; sg < nsg; ++sg) {
      f2_mbar_wait(&rg.full[rg.rs], rg.rph);
      const double* stage = rg.ring + (size_t)rg.rs * F2_STG;
#pragma unroll
      for (int sub = 0; sub < F2_SBS; ++sub) {
        const double* tile = stage + (size_t)sub * 8 * F2_TS;
        const int sb = sg * F2_SBS + sub;
        // all fragment loads of the series block first (no branches in between: the warp issues in order, so a
        // load placed after a DMMA would only start once that DMMA's operands had arrived), then the math
        double lm[2], av[2][F2_NRB];
#pragma unroll
        for (int kc = 0; kc < 2; ++kc) {
          const int n = sb * 8 + kc * 4 + lc;
          const bool nok = n < N;
          lm[kc] = (nok && lr < R) ? W[LI(n, lr)] : 0.0;
          const double* trow = tile + (kc * 4 + lc) * F2_TS + lr;
#pragma unroll
          for (int j = 0; j < F2_NRB; ++j) {
            const int t0 = (cw + j * F2_NCW) * 8;
            av[kc][j] = (nok && t0 + lr < len) ? trow[t0] : 0.0;
          }
        }
#pragma unroll
        for (int kc = 0; kc < 2; ++kc)
#pragma unroll
          for (int j = 0; j < F2_NRB; ++j) {
            if (SQ) qacc += av[kc][j] * av[kc][j];
            asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
                         : "+d"(d[j][kc][0]), "+d"(d[j][kc][1]) : "d"(av[kc][j]), "d"(lm[kc]));
          }
      }
      __syncwarp();
      if (lane == 0) f2_mbar_arrive(&rg.empty[rg.rs]);
      rg.advance();
    }
#pragma unroll
    for (int j = 0; j < F2_NRB; ++j) {
      const int tl = (cw + j * F2_NCW) * 8 + lr;
      if (tl < len) { const int t = c * F2_TC + tl; Z[ZI(t, 2 * lc)] = d[j][0][0] + d[j][1][0]; Z[ZI(t, 2 * lc + 1)] = d[j][0][1] + d[j][1][1]; }
    }
  }
  return qacc;
}

// M pass, consumer warp cw:  Lam[n][:] <- sum_t x[t,n] Z[t][:]  (S_xf) and, if FIRST, sxx[n] <- sum_t x[t,n]^2
// (the same in every iteration: later passes leave sxx alone and reduce 64 values per series block instead of 72).
// Series-block outer in descending order (f2_produce) / period-chunk inner; two accumulator pairs per warp;
// deterministic cross-warp reduction of the F2_NCW partial tiles at the end of every series block (named barrier 1).
// A block's sums depend on its own chunks only, so the block order does not change any result.
template <int R, bool FIRST>
__device__ __forceinline__ void f2_consume_M(F2Ring& rg, int cw, int T, int N, int Tp, int Np, const double* Z, double* Lam,
                                             double* sxx, double* part) {
  const int lane = threadIdx.x & 31, lr = lane >> 2, lc = lane & 3;
  const int nsg = (N + 8 * F2_SBS - 1) / (8 * F2_SBS), nck = (T + F2_TC - 1) / F2_TC;
  // one accumulator pair per (series block of the stage, k-chunk slot): independent DMMAs
  double d[F2_SBS][F2_NKC][2], s2[F2_SBS];
#pragma unroll
  for (int sub = 0; sub < F2_SBS; ++sub) {
    s2[sub] = 0.0;
#pragma unroll
    for (int j = 0; j < F2_NKC; ++j) { d[sub][j][0] = 0.0; d[sub][j][1] = 0.0; }
  }
  for (int sg = nsg - 1; sg >= 0; --sg)
    for (int c = 0; c < nck; ++c) {
      f2_mbar_wait(&rg.full[rg.rs], rg.rph);
      const double* stage = rg.ring + (size_t)rg.rs * F2_STG;
      const int len = (T - c * F2_TC < F2_TC) ? T - c * F2_TC : F2_TC;
      const double* zc = Z + (size_t)lr * Tp + c * F2_TC + lc;
      double bv[F2_NKC];                                         // Z fragments: shared by the series blocks of the stage
#pragma unroll
      for (int j = 0; j < F2_NKC; ++j) { const int t0 = (cw + j * F2_NCW) * 4; bv[j] = (t0 + lc < len) ? zc[t0] : 0.0; }
#pragma unroll
      for (int sub = 0; sub < F2_SBS; ++sub) {
        const bool nok = (sg * F2_SBS + sub) * 8 + lr < N;
        const double* trow = stage + (size_t)sub * 8 * F2_TS + lr * F2_TS + lc;
        double av[F2_NKC];                                       // k-chunks cw, cw + NCW, ...: loads first, then the math
#pragma unroll
        for (int j = 0; j < F2_NKC; ++j) { const int t0 = (cw + j * F2_NCW) * 4; av[j] = (nok && t0 + lc < len) ? trow[t0] : 0.0; }
#pragma unroll
        for (int j = 0; j < F2_NKC; ++j) {
          if (FIRST) s2[sub] += av[j] * av[j];
          asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
                       : "+d"(d[sub][j][0]), "+d"(d[sub][j][1]) : "d"(av[j]), "d"(bv[j]));
        }
      }
      __syncwarp();
      if (lane == 0) f2_mbar_arrive(&rg.empty[rg.rs]);
      rg.advance();
      if (c == nck - 1) {
        // cross-warp reduction of the F2_NCW partial tiles, one series block after the other; buffer = block parity
        // (a block's partials are rewritten two barriers later at the earliest)
#pragma unroll
        for (int sub = 0; sub < F2_SBS; ++sub) {
          const int sb = sg * F2_SBS + sub;
          double* pb = part + (size_t)(sb & 1) * F2_NCW * 72 + cw * 72;
          double t0_ = 0.0, t1_ = 0.0;
#pragma unroll
          for (int j = 0; j < F2_NKC; ++j) { t0_ += d[sub][j][0]; t1_ += d[sub][j][1]; d[sub][j][0] = 0.0; d[sub][j][1] = 0.0; }
          pb[2 * lane] = t0_; pb[2 * lane + 1] = t1_;
          if (FIRST) {
            double sq = s2[sub];
            sq += __shfl_xor_sync(0xffffffffu, sq, 1); sq += __shfl_xor_sync(0xffffffffu, sq, 2);
            if (lc == 0) pb[64 + lr] = sq;
          }
          asm volatile("bar.sync 1, %0;" ::"n"(F2_NCW * 32) : "memory");
          const int ct = cw * 32 + lane;                          // 0 .. F2_NCW*32-1
          if (ct < (FIRST ? 72 : 64)) {
            const double* pp_ = part + (size_t)(sb & 1) * F2_NCW * 72 + ct;
            double tot_ = 0.0;
#pragma unroll
            for (int w_ = 0; w_ < F2_NCW; ++w_) tot_ += pp_[w_ * 72];
            if (ct < 64) {
              const int l_ = ct >> 1, h_ = ct & 1, row = l_ >> 2, col = 2 * (l_ & 3) + h_, n = sb * 8 + row;
              if (n < N && col < R) Lam[LI(n, col)] = tot_;
            } else { const int n = sb * 8 + (ct - 64); if (n < N) sxx[n] = tot_; }
          }
          s2[sub] = 0.0;
        }
      }
    }
}
#endif  // !DFM_EMU

// the mean recursions P3-P5 run on warps 0..F2_NCW (named barrier 2) while the chain warp does the backward covariances
#define F2_PNT_GPU ((F2_NCW + 1) * 32)
#ifdef DFM_EMU
#define F2_PSYNC() ((void)0)
#define F2_PTID 0
#define F2_PNT 1
#else
#define F2_PSYNC() asm volatile("bar.sync 2, %0;" ::"n"(F2_PNT_GPU) : "memory")
#define F2_PTID ((int)threadIdx.x)
#define F2_PNT F2_PNT_GPU
#endif
#ifdef DFM_EMU
#define DFM_FUSED2_BOUNDS
#else
#define DFM_FUSED2_BOUNDS __launch_bounds__(256, 2)
#endif
template <int R>
__global__ void DFM_FUSED2_BOUNDS k_em_fused2(FusedArgs a, const DFM_GRID_CONSTANT CUtensorMap tmap) {
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
  double* scal = red + 40;                 // 8: [0]=slr [1]=ld_inf [2]=sum x'R^-1 x [3]=ll
  int* ctl = (int*)(scal + 8);             // [0]=nE [1]=tb [2]=bad [3]=frozen [4]=turn window of the panel (f2_produce)
  double* bnd = scal + 16;                 // (3*32+1) R + RR: blk_recur workspace for 32 groups
  double* part = bnd;                                // [2][F2_NCW][72] M-pass partial accumulators: ALIASES the scan
                                                     // workspace (used only inside the M pass / only in P3, P5)
  double* ring = bnd + (((size_t)97 * R + RR > 2 * F2_NCW * 72) ? (size_t)97 * R + RR : 2 * F2_NCW * 72);   // F2_S stages x 8 x F2_TS
#ifndef DFM_EMU
  ring += ((128u - (f2_smem_u32(ring) & 127u)) & 127u) / 8;      // tensor-map copies need 128-byte aligned destinations
#endif
  double* gscr = a.scratch + (size_t)DFM_BX * T * FUSED_SCR(R);
  // per explicit step t: SCRP(t)[{0:Pf, RR:Phi, 2RR:J, 3RR:W, 4RR:Ps, 5RR: ld}]; the first F2_NEXS(R)
  // steps live in the (idle between the two passes) ring, the rest in global scratch
#define GSC(t_) (gscr + (size_t)(t_) * FUSED_SCR(R))
#define SCRP(t_) (((t_) < F2_NEXS(R)) ? (ring + (size_t)(t_) * FUSED_SCR(R)) : (gscr + (size_t)(t_) * FUSED_SCR(R)))
#define GPS(t_) (gscr + (size_t)(t_) * FUSED_SCR(R) + 4 * RR)      // smoothed covariances: always global (read at output time only)
#ifndef DFM_EMU
  __shared__ uint64_t fullb[F2_S], emptyb[F2_S];
  if (threadIdx.x == 0) { for (int s_ = 0; s_ < F2_S; ++s_) { f2_mbar_init(&fullb[s_], 1); f2_mbar_init(&emptyb[s_], F2_NCW); } }
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  __syncthreads();
  F2Ring rg; rg.ring = ring; rg.full = fullb; rg.empty = emptyb; rg.rs = 0; rg.rph = 0; rg.wrap = false;
#endif
  const double eps = 1e-14;

  for (int b = DFM_BX; b < a.B; b += DFM_GX) {
#ifdef DFM_EMU
    const double* X = a.X + (size_t)b * T * N;
#endif
#ifndef DFM_EMU
    if (a.ready) {                             // streaming host path: wait until this panel's chunk has landed
      if (threadIdx.x == 0) {
        const int* f_ = a.ready + b / a.ready_chunk; int v_ = 0;
        for (;;) { asm volatile("ld.acquire.sys.global.s32 %0, [%1];" : "=r"(v_) : "l"(f_) : "memory"); if (v_) break; __nanosleep(256); }
      }
      __syncthreads();
    }
#endif
    // ---- load parameters (global column-major -> shared row-major)
    for (int e = DFM_TID; e < N * R; e += DFM_NT) { int i = e % N, c = e / N; Lam[LI(i, c)] = a.Lam[(size_t)b * N * R + e]; }
    for (int e = DFM_TID; e < N; e += DFM_NT) Rv[e] = a.R[(size_t)b * N + e];
    for (int e = DFM_TID; e < RR; e += DFM_NT) {
      int i = e / R, j = e % R;
      M[e] = a.A[(size_t)b * RR + i + R * j]; Q[e] = a.Q[(size_t)b * RR + i + R * j];
    }
    if (DFM_TID == 0) ctl[2] = 0;
#ifndef DFM_EMU
    if (DFM_TID == 0) ctl[4] = f2_round_win(a.l2_win, a.B, b);
#endif
    DFM_SYNC();
    if (a.P0out || a.ready) {
      // initial state covariance in the kernel: P0 = sum_i A^i Q A'^i by doubling (same recursion as k_lyapunov), on
      // the first RR threads; Pp = P, Pi = A^(2^s).  This panel's log-likelihood row is pre-filled here as well.
      for (int e = DFM_TID; e < a.max_iter; e += DFM_NT) a.loglik[(size_t)b * a.max_iter + e] = DFM_NAN;
      if (a.P0out) {
        // plain sequential dot products in the order of k_lyapunov / bm_gemm: bit-identical P0 on both host paths
        for (int e = DFM_TID; e < RR; e += DFM_NT) { Pp[e] = Q[e]; Pi[e] = M[e]; }
        DFM_SYNC();
        for (int s_ = 0; s_ < a.p0_steps; ++s_) {
          for (int e = DFM_TID; e < RR; e += DFM_NT) { const int i = e / R, j = e % R; double v = 0.0; for (int l = 0; l < R; ++l) v += Pi[i * R + l] * Pp[l * R + j]; Wm[e] = v; }
          DFM_SYNC();
          for (int e = DFM_TID; e < RR; e += DFM_NT) { const int i = e / R, j = e % R; double v = 0.0; for (int l = 0; l < R; ++l) v += Wm[i * R + l] * Pi[j * R + l]; G[e] = v; }
          DFM_SYNC();
          for (int e = DFM_TID; e < RR; e += DFM_NT) {
            const int i = e / R, j = e % R; double v = 0.0; for (int l = 0; l < R; ++l) v += Pi[i * R + l] * Pi[l * R + j];
            Wm[e] = v; Pp[e] = Pp[e] + 1.0 * G[e];
          }
          DFM_SYNC();
          for (int e = DFM_TID; e < RR; e += DFM_NT) Pi[e] = Wm[e];
          DFM_SYNC();
        }
        for (int e = DFM_TID; e < RR; e += DFM_NT) { const int i = e / R, j = e % R; if (i > j) { const double v = 0.5 * (Pp[i * R + j] + Pp[j * R + i]); Pp[i * R + j] = v; Pp[j * R + i] = v; } }
        DFM_SYNC();
        for (int e = DFM_TID; e < RR; e += DFM_NT) { const int i = e / R, j = e % R; a.P0out[(size_t)b * RR + i + R * j] = Pp[e]; }
      }
      DFM_SYNC();                                  // (the chain warp reads a.P0 == a.P0out of this panel from global)
    }
    int it = 0, status = 0;
    double ll_prev = 0.0;
    for (; it < a.max_iter; ++it) {
      // ---------------------------------------------------------------- P0: prep
      // sum log R and, from the second iteration on (the first M pass fills sxx), sum x'R^-1 x = sum_n sxx_n / R_n
      double slr_p = 0.0, q_p = 0.0;
      for (int i = DFM_TID; i < N; i += DFM_NT) {
        const double rv = Rv[i], ri = 1.0 / rv;
        rinv[i] = ri; slr_p += log(rv); if (it > 0) q_p += sxx[i] * ri;
        if (!(rv > 0.0)) ctl[2] = 1;
      }
      slr_p = block_sum(slr_p, red);
      if (it > 0) q_p = block_sum(q_p, red);
      if (DFM_TID == 0) { scal[0] = slr_p; scal[2] = q_p; }
      DFM_SYNC();
      {   // C = Lam' R^-1 Lam: RR outputs x (NT / RR) slices of the series range, combined in fixed order
        const int nsl = (DFM_NT >= 4 * RR) ? 4 : 1;
#ifndef DFM_EMU
        if (R == 8) {
          // tensor path: C = (Lam .* rinv)' Lam as DMMA.8x8x4 over 4-series chunks; the B fragment is the Lam value the
          // A fragment is built from.  Warps 0..3 produce the nsl = 4 partial tiles (chunks w, w+4, w+8, ...).
          if (DFM_WARP < 4) {
            const int lr = DFM_LANE >> 2, lc = DFM_LANE & 3;
            const double* lrow = Lam + (size_t)lr * Np;
            double c0 = 0.0, c1 = 0.0, e0 = 0.0, e1 = 0.0;
            for (int ch = DFM_WARP; 4 * ch < N; ch += 8) {
              const int na = 4 * ch + lc, nb = 4 * (ch + 4) + lc;
              const double la = (na < N) ? lrow[na] : 0.0, ra = (na < N) ? rinv[na] : 0.0;
              const double lb = (nb < N) ? lrow[nb] : 0.0, rb = (nb < N) ? rinv[nb] : 0.0;
              const double aa = la * ra, ab = lb * rb;
              asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n" : "+d"(c0), "+d"(c1) : "d"(aa), "d"(la));
              asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n" : "+d"(e0), "+d"(e1) : "d"(ab), "d"(lb));
            }
            T1[DFM_WARP * RR + 2 * DFM_LANE] = c0 + e0; T1[DFM_WARP * RR + 2 * DFM_LANE + 1] = c1 + e1;
          }
        } else
#endif
        for (int e = DFM_TID; e < nsl * RR; e += DFM_NT) {
          int sl = e / RR, ee = e % RR, i = ee / R, j = ee % R;
          int n0 = (int)((long long)N * sl / nsl), n1 = (int)((long long)N * (sl + 1) / nsl);
          double s = 0.0;
          for (int n = n0; n < n1; ++n) s += Lam[LI(n, i)] * rinv[n] * Lam[LI(n, j)];
          T1[sl * RR + ee] = s;                    // T1, T2, Ps, Psn are contiguous scratch matrices
        }
        DFM_SYNC();
        for (int e = DFM_TID; e < RR; e += DFM_NT) { double s = 0.0; for (int sl = 0; sl < nsl; ++sl) s += T1[sl * RR + e]; C[e] = s; }
        // the E pass contracts with W = R^-1 Lam: scale the loadings in place.  Nothing reads them as Lam again before
        // the M pass overwrites them with S_xf, and the loop exits only after P9 has written the new Lam.
        for (int e = DFM_TID; e < N * R; e += DFM_NT) { const int n = e % N, c = e / N; Lam[LI(n, c)] *= rinv[n]; }
      }
      DFM_SYNC();
      // ---- covariance chain (data independent).  Forward part: on the chain warp concurrently with the E pass;
      //      backward part (smoothed covariances + covariance parts of the moment sums): on the chain warp
      //      concurrently with the mean recursions P3-P5, which only need the forward quantities (Pf, Phi, J).
      auto chain_fwd = [&]() {
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
          double* s_ = GSC(t);
          double dmax = 0.0, pmax = 0.0;
          for (int e = DFM_LANE; e < RR; e += DFM_WSZ) {
            s_[e] = Pf[e]; s_[RR + e] = Phi[e]; s_[3 * RR + e] = Wm[e];
            if (t >= 1) GSC(t - 1)[2 * RR + e] = Jm[e];
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
        if (DFM_LANE == 0) { ctl[0] = nE; ctl[3] = frozen; }
        // I - J_inf M  (for the parallel pre-pass of the backward mean recursion)
        if (frozen) {
          w_gemm<R>(IJM, Jinf, false, M, false);
          for (int e = DFM_LANE; e < RR; e += DFM_WSZ) { int i = e / R, j = e % R; IJM[e] = ((i == j) ? 1.0 : 0.0) - IJM[e]; }
          DFM_WSYNC();
          // chunk-length powers of the two scan matrices (P3: Phi_inf, P5: J_inf), off the critical path of P3/P5.
          // Phi and Pn are free from here until the M-step solves; T1/T2 serve as scratch.
          const int n3 = T - (nE > 0 ? nE : 1), n5 = (T - 2) - (nE - 1) + 1;
          if (n3 > 0) {
            w_matpow<R>(Phi, Phinf, blk_chunk_len(n3, F2_PNT_GPU / 8), T1, T2);
            // Kogge-Stone levels of the forward scan: (Phi^Lc)^2, ^4, ^8, ^16 in forward-chain temporaries that are idle now
            w_gemm<R>(Pp, Phi, false, Phi, false); w_gemm<R>(Pi, Pp, false, Pp, false);
            w_gemm<R>(Pf, Pi, false, Pi, false);   w_gemm<R>(Jm, Pf, false, Pf, false);
          }
          if (n5 > 0) {
            w_matpow<R>(Pn, Jinf, blk_chunk_len(n5, F2_PNT_GPU / 8), T1, T2);
            // ... of the backward scan: parked in the unused slots of the last scratch entry (the ring is busy with
            // the E pass), copied into the ring tail together with the explicit steps
            double* gl_ = GSC(T - 1);
            w_gemm<R>(T1, Pn, false, Pn, false);
            for (int e = DFM_LANE; e < RR; e += DFM_WSZ) gl_[e] = T1[e];
            w_gemm<R>(T2, T1, false, T1, false);
            for (int e = DFM_LANE; e < RR; e += DFM_WSZ) gl_[RR + e] = T2[e];
            w_gemm<R>(T1, T2, false, T2, false);
            for (int e = DFM_LANE; e < RR; e += DFM_WSZ) gl_[2 * RR + e] = T1[e];
            w_gemm<R>(T2, T1, false, T1, false);
            for (int e = DFM_LANE; e < RR; e += DFM_WSZ) gl_[3 * RR + e] = T2[e];
            DFM_WSYNC();
          }
        }
        DFM_WSYNC();
      };
      auto chain_bwd = [&]() {
        const int nE = ctl[0], frozen = ctl[3];
        int t;
        // backward covariance chain + covariance parts of the moment sums
        for (int e = DFM_LANE; e < RR; e += DFM_WSZ) {
          double v = frozen ? Pfinf[e] : (GSC(T - 1))[e];
          Psn[e] = v; SPall[e] = v; SPff2[e] = v; SP00[e] = 0.0; SP11[e] = 0.0;
          GPS(T - 1)[e] = v;
        }
        DFM_WSYNC();
        const int lo = frozen ? nE - 1 : T;
        int tb = -1;                        // frozen smoothed range is [lo, tb)
        t = T - 2;
        while (t >= 0) {
          const double* pf_t = (t < nE) ? GSC(t) : Pfinf;
          const double* j_t = (t < nE - 1) ? GSC(t) + 2 * RR : Jinf;
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
            GPS(t)[e] = Ps[e];
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
        if (DFM_LANE == 0) ctl[1] = tb;
        DFM_WSYNC();
      };
      // ---------------------------------------------------------------- P1: E-step contraction (panel pass 1)
      //   b_t = W' x_t  (W = R^-1 Lam); the data term -1/2 sum x'R^-1 x of the log-likelihood comes from sxx (P0, P9)
#ifdef DFM_EMU
      for (int t = 0; t < T; ++t) {
        for (int c = 0; c < FZ; ++c) Z[ZI(t, c)] = 0.0;
        for (int n = 0; n < N; ++n) {
          double x = X[(size_t)n * T + t];
          for (int c = 0; c < R; ++c) Z[ZI(t, c)] += x * Lam[LI(n, c)];
        }
      }
#else
      {
        // TMA pass (see f2_produce / f2_consume_E): warp 0 produces, warps 1..6 consume, warp 7 runs the
        // data-independent covariance chain concurrently
        const long long nitems = (long long)((N + 8 * F2_SBS - 1) / (8 * F2_SBS)) * ((T + F2_TC - 1) / F2_TC);
        if (DFM_WARP == 0) f2_produce(rg, &tmap, b * N, T, N, /*c_outer=*/true, &ctl[4]);
        else if (DFM_WARP <= F2_NCW) f2_consume_E<R, false>(rg, DFM_WARP - 1, T, N, Tp, Np, Z, Lam);
        else {
          rg.skip(nitems);                                                   // keep the ring position in step
          chain_fwd();
        }
      }
#endif
#ifdef DFM_EMU
      chain_fwd();
      chain_bwd();
#endif
      DFM_SYNC();                                            // E pass and forward chain complete
      const int nE = ctl[0], frozen = ctl[3];
#ifndef DFM_EMU
      if (DFM_WARP == F2_NCW + 1) chain_bwd();                 // warp 7: backward covariance chain, concurrently with P3-P5 on warps 0..6
      else
#endif
      {
      {   // explicit covariance steps: global scratch -> (now idle) ring, one cooperative copy; first read after
          // the barrier that follows the pre-pass below
        const int ncp = (nE < F2_NEXS(R)) ? nE : F2_NEXS(R);
        for (int e = F2_PTID; e < ncp * FUSED_SCR(R); e += F2_PNT) ring[e] = gscr[e];
        if (frozen) for (int e = F2_PTID; e < 4 * RR; e += F2_PNT) ring[F2_RTAIL(R) + e] = GSC(T - 1)[e];   // backward-scan level matrices
      }
      // ---------------------------------------------------------------- P3: forward means
      // parallel pre-pass over the frozen range: Z[t] <- Pf_inf b_t
      for (int t = nE + F2_PTID; t < T; t += F2_PNT) {
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
      F2_PSYNC();
      if (DFM_WARP == 0) {
        // explicit steps
        for (int t = 0; t < nE; ++t) {
          const double* s_ = SCRP(t);
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
      F2_PSYNC();
      // frozen steps: z_t = Phi_inf z_{t-1} + u_t, parallel in time over the CTA
      if (frozen) blk_recur<R>(Z, Tp, Phinf, Phi, Pi, bnd, (nE > 0 ? nE : 1), T - (nE > 0 ? nE : 1), +1, F2_PNT_GPU, true, Pp, Pi, Pf, Jm);
      // ---------------------------------------------------------------- P4: log-likelihood
      // innovation form: ll_t = -1/2 (N log 2pi + sum log R + ld_t + quad_t),
      //   quad_t = -(zp'C zp + 2 zp'W d + d'W d),  zp = M zf_{t-1}, d = zf_t - zp,  W = Pi + C
      // which collapses to  quad_t = zf_{t-1}' K zf_{t-1} - zf_t' W zf_t  with K = M'(W - C) M.  Over the frozen
      // range (W, K constant) the sum only needs the second-moment matrix of the filtered means:
      //   sum_t quad_t = tr(K (Gf + z_{nE-1} z_{nE-1}' - z_{T-1} z_{T-1}')) - tr(W Gf),   Gf = sum_{t>=nE} zf_t zf_t'.
      // plus the data term -1/2 sum x'R^-1 x (P0), on one thread; the first iteration's is added in P9
      double llp = (it > 0 && F2_PTID == 0) ? -0.5 * scal[2] : 0.0;
      const bool gram = frozen && nE >= 1 && nE < T;
      // explicit periods t < nE: one thread per (t, component) in two stages when their (zp, d) vectors fit
      // in the idle scan workspace; otherwise (and for a chain that never froze) one thread per period
      const bool split = gram && 2 * nE * R <= (97 * R + RR) - (F2_GPARTS + 1) * RR;
      const int tex = gram ? (split ? 0 : nE) : T;           // periods handled one thread each
      if (gram) {
        double* gp = bnd;                                    // [F2_GPARTS][RR] partial Gram sums, then K (scan workspace is idle)
#ifndef DFM_EMU
        if (R == 8) {
          // Gram matrix on the FP64 tensor path: D[8x8] += Zc Zc' for 4-period chunks; the A and the B fragment of
          // DMMA.8x8x4 are the same register (A[i][k] = B[k][i] = z_i(t0 + k)); warp w takes chunks w, w+7, ...
          const int lr = DFM_LANE >> 2, lc = DFM_LANE & 3;
          const double* zr = Z + (size_t)lr * Tp;
          double g0 = 0.0, g1 = 0.0, h0 = 0.0, h1 = 0.0;
          for (int t0 = nE + 4 * DFM_WARP; t0 < T; t0 += 8 * (F2_NCW + 1)) {
            const int ta = t0 + lc, tb_ = t0 + 4 * (F2_NCW + 1) + lc;
            const double va = (ta < T) ? zr[ta] : 0.0, vb = (tb_ < T) ? zr[tb_] : 0.0;
            asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n" : "+d"(g0), "+d"(g1) : "d"(va), "d"(va));
            asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n" : "+d"(h0), "+d"(h1) : "d"(vb), "d"(vb));
          }
          gp[DFM_WARP * 64 + 2 * DFM_LANE] = g0 + h0; gp[DFM_WARP * 64 + 2 * DFM_LANE + 1] = g1 + h1;     // element (lr, 2 lc), (lr, 2 lc + 1)
        } else
#endif
        {
          const int nfz = T - nE, q4 = (nfz + F2_GPARTS_S - 1) / F2_GPARTS_S;
          for (int e = F2_PTID; e < F2_GPARTS * RR; e += F2_PNT) {
            const int q = e / RR, ee = e % RR, i = ee / R, jj = ee % R;
            double s0_ = 0.0, s1_ = 0.0;
            if (q < F2_GPARTS_S) {
              const int lo = nE + q * q4, hi = (lo + q4 < T) ? lo + q4 : T;
              int t = lo;
              for (; t + 1 < hi; t += 2) { s0_ += Z[ZI(t, i)] * Z[ZI(t, jj)]; s1_ += Z[ZI(t + 1, i)] * Z[ZI(t + 1, jj)]; }
              if (t < hi) s0_ += Z[ZI(t, i)] * Z[ZI(t, jj)];
            }
            gp[e] = s0_ + s1_;
          }
        }
        if (split) {                                         // stage A: zp = M zf_{t-1}, d = zf_t - zp
          double* zd = gp + (F2_GPARTS + 1) * RR;
          for (int e = F2_PTID; e < nE * R; e += F2_PNT) {
            const int t = e / R, i = e % R;
            double s_ = 0.0;
            if (t >= 1) {
#pragma unroll
              for (int j = 0; j < R; ++j) s_ += M[i * R + j] * Z[ZI(t - 1, j)];
            }
            zd[2 * e] = s_; zd[2 * e + 1] = Z[ZI(t, i)] - s_;
          }
        }
        if (DFM_WARP == 0) {                                 // K = M'(W_inf - C) M on warp 0 meanwhile (T2 = W - C, T1 = T2 M)
          for (int e = DFM_LANE; e < RR; e += DFM_WSZ) Wm[e] = Winf[e] - C[e];     // (Wm, G: forward-chain temporaries, idle now;
          DFM_WSYNC();                                                             //  T1/T2 belong to the backward chain on warp 7)
          w_gemm<R>(G, Wm, false, M, false);
          w_gemm<R>(gp + F2_GPARTS * RR, M, true, G, false);
        }
        F2_PSYNC();
        for (int e = F2_PTID; e < RR; e += F2_PNT) {
          const int i = e / R, jj = e % R;
          double gf = 0.0;
#pragma unroll
          for (int q = 0; q < F2_GPARTS; ++q) gf += gp[q * RR + e];
          const double gs = gf + Z[ZI(nE - 1, i)] * Z[ZI(nE - 1, jj)] - Z[ZI(T - 1, i)] * Z[ZI(T - 1, jj)];
          llp += -0.5 * (gp[F2_GPARTS * RR + e] * gs - Winf[e] * gf);
        }
        if (F2_PTID == 0) llp += -0.5 * (double)(T - nE) * ((double)N * 1.8378770664093454835606594728112 + scal[0] + scal[1]);
        if (split) {                                         // stage B: row i of  zp'C zp + 2 zp'W_t d + d'W_t d
          const double* zd = gp + (F2_GPARTS + 1) * RR;
          for (int e = F2_PTID; e < nE * R; e += F2_PNT) {
            const int t = e / R, i = e % R;
            const double* Wt = SCRP(t) + 3 * RR;
            const double* zt = zd + 2 * (size_t)t * R;
            double cz = 0.0, g = 0.0;
#pragma unroll
            for (int j = 0; j < R; ++j) { cz += C[i * R + j] * zt[2 * j]; g += Wt[i * R + j] * zt[2 * j + 1]; }
            const double zpi = zt[2 * i], di = zt[2 * i + 1];
            llp += 0.5 * (zpi * cz + 2.0 * zpi * g + g * di);
            if (i == 0) llp += -0.5 * ((double)N * 1.8378770664093454835606594728112 + scal[0] + (SCRP(t))[5 * RR]);
          }
        }
      }
      for (int t = F2_PTID; t < tex; t += F2_PNT) {
        const double* Wt = (t < nE) ? SCRP(t) + 3 * RR : Winf;
        double ldt = (t < nE) ? (SCRP(t))[5 * RR] : scal[1];
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
      {   // sum over the F2_PNT threads of this section (fixed order), result in scal[3]
#ifndef DFM_EMU
        for (int o = 16; o > 0; o >>= 1) llp += __shfl_down_sync(0xffffffffu, llp, o);
        if (DFM_LANE == 0) red[DFM_WARP] = llp;
        F2_PSYNC();
        if (threadIdx.x == 0) { double s_ = 0.0; for (int w_ = 0; w_ <= F2_NCW; ++w_) s_ += red[w_]; scal[3] = s_; }
#else
        scal[3] = llp;
#endif
      }
      // ---------------------------------------------------------------- P5: backward means
      if (frozen) {
        int lo = nE - 1;
        for (int t = lo + F2_PTID; t < T - 1; t += F2_PNT) {       // Z[t] <- (I - J_inf M) zf_t
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
      F2_PSYNC();
      // frozen range: z_t = J_inf z_{t+1} + v_t, parallel in time over the CTA
      if (frozen) blk_recur<R>(Z, Tp, Jinf, Pn, Pi, bnd, T - 2, (T - 2) - (nE - 1) + 1, -1, F2_PNT_GPU, true, ring + F2_RTAIL(R), ring + F2_RTAIL(R) + RR, ring + F2_RTAIL(R) + 2 * RR, ring + F2_RTAIL(R) + 3 * RR);
      if (DFM_WARP == 0) {
        const int lo = frozen ? nE - 1 : T;
        // explicit range: zs_t = zf_t + J_t (zs_{t+1} - M zf_t)
        for (int t = (lo - 1 < T - 2 ? lo - 1 : T - 2); t >= 0; --t) {
          const double* j_t = SCRP(t) + 2 * RR;
          for (int i = DFM_LANE; i < R; i += DFM_WSZ) { double s = Z[ZI(t + 1, i)]; for (int j = 0; j < R; ++j) s -= M[i * R + j] * Z[ZI(t, j)]; tmp[i] = s; }
          DFM_WSYNC();
          for (int i = DFM_LANE; i < R; i += DFM_WSZ) { double s = Z[ZI(t, i)]; for (int j = 0; j < R; ++j) s += j_t[i * R + j] * tmp[j]; tmp[R + i] = s; }
          DFM_WSYNC();
          for (int i = DFM_LANE; i < R; i += DFM_WSZ) Z[ZI(t, i)] = tmp[R + i];
          DFM_WSYNC();
        }
      }
      }
      DFM_SYNC();
      // ---- moment sums + M-step r x r solves (all inputs are ready before the M pass): on the chain warp,
      //      concurrently with the pass
      auto mstep_small = [&]() {
        int* bad = &ctl[2];
        // mean parts of the moment sums (needs only the smoothed means in Z)
#ifndef DFM_EMU
        if (R == 8) {
          // Sm = sum_t z_t z_t' and S11m = sum_{t>=1} z_t z_{t-1}' as DMMA.8x8x4 Gram products over 4-period chunks: the A
          // fragment (z_i(t0 + k)) doubles as the B fragment of Sm; S11m takes z_j(t0 + k - 1) as B.  Two accumulator
          // pairs each (chunks alternate), ~2 x 125 DMMAs instead of 2 x 64 x T scalar multiply-adds on 32 lanes
          // (chain-warp time in the M pass: 12.1M -> 5.5M cycles per CTA).
          const int lr = DFM_LANE >> 2, lc = DFM_LANE & 3;
          const double* zr = Z + (size_t)lr * Tp;
          double g[2][2] = {{0.0, 0.0}, {0.0, 0.0}}, h[2][2] = {{0.0, 0.0}, {0.0, 0.0}};
          for (int t0 = 0; t0 < T; t0 += 8) {
            const int ta = t0 + lc, tb_ = t0 + 4 + lc;
            const double va = (ta < T) ? zr[ta] : 0.0, vb = (tb_ < T) ? zr[tb_] : 0.0;
            const double pa = (ta >= 1 && ta < T) ? zr[ta - 1] : 0.0, pb = (tb_ < T) ? zr[tb_ - 1] : 0.0;
#define F2_DMMA(d_, a_, b_) asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n" : "+d"((d_)[0]), "+d"((d_)[1]) : "d"(a_), "d"(b_))
            F2_DMMA(g[0], va, va); F2_DMMA(h[0], va, pa);
            F2_DMMA(g[1], vb, vb); F2_DMMA(h[1], vb, pb);
#undef F2_DMMA
          }
          Sm[lr * 8 + 2 * lc] = g[0][0] + g[1][0]; Sm[lr * 8 + 2 * lc + 1] = g[0][1] + g[1][1];
          S11m[lr * 8 + 2 * lc] = h[0][0] + h[1][0]; S11m[lr * 8 + 2 * lc + 1] = h[0][1] + h[1][1];
        } else
#endif
        for (int e = DFM_LANE; e < 2 * RR; e += DFM_WSZ) {
          int which = e / RR, ee = e % RR, i = ee / R, j = ee % R;
          double s0 = 0.0, s1 = 0.0;
          if (which == 0) { for (int t = 0; t + 1 < T; t += 2) { s0 += Z[ZI(t, i)] * Z[ZI(t, j)]; s1 += Z[ZI(t + 1, i)] * Z[ZI(t + 1, j)]; }
                            if (T & 1) s0 += Z[ZI(T - 1, i)] * Z[ZI(T - 1, j)]; Sm[ee] = s0 + s1; }
          else { for (int t = 1; t + 1 < T; t += 2) { s0 += Z[ZI(t, i)] * Z[ZI(t - 1, j)]; s1 += Z[ZI(t + 1, i)] * Z[ZI(t, j)]; }
                 if (!(T & 1)) s0 += Z[ZI(T - 1, i)] * Z[ZI(T - 2, j)]; S11m[ee] = s0 + s1; }
        }
        DFM_WSYNC();

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
      };
      // ---------------------------------------------------------------- P8: M-step contraction (panel pass 2)
#ifdef DFM_EMU
      for (int n = 0; n < N; ++n) {
        double s2 = 0.0, acc[R];
        for (int c = 0; c < R; ++c) acc[c] = 0.0;
        for (int t = 0; t < T; ++t) { double x = X[(size_t)n * T + t]; if (it == 0) s2 += x * x; for (int c = 0; c < R; ++c) acc[c] += x * Z[ZI(t, c)]; }
        for (int c = 0; c < R; ++c) Lam[LI(n, c)] = acc[c];
        if (it == 0) sxx[n] = s2;
      }
#else
      {
        // the ring held explicit-step scratch written with ordinary stores: order them before the
        // async-proxy writes of the bulk copies
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        __syncthreads();
        const long long nitems = (long long)((N + 8 * F2_SBS - 1) / (8 * F2_SBS)) * ((T + F2_TC - 1) / F2_TC);
        if (DFM_WARP == 0) f2_produce(rg, &tmap, b * N, T, N, /*c_outer=*/false, &ctl[4]);
        else if (DFM_WARP <= F2_NCW) {
          if (it == 0) f2_consume_M<R, true>(rg, DFM_WARP - 1, T, N, Tp, Np, Z, Lam, sxx, part);
          else f2_consume_M<R, false>(rg, DFM_WARP - 1, T, N, Tp, Np, Z, Lam, nullptr, part);
        } else {
          rg.skip(nitems);
          mstep_small();
        }
      }
#endif
#ifdef DFM_EMU
      mstep_small();
#endif
      DFM_SYNC();
      // ---------------------------------------------------------------- P9: M-step solves
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
      // the data term of the first iteration's log-likelihood, now that its M pass has filled sxx (P0, P4: later ones)
      double xrx = 0.0;
      if (it == 0 && DFM_TID == 0) { for (int n = 0; n < N; ++n) xrx += sxx[n] * rinv[n]; }
      DFM_SYNC();
      if (it == 0 && DFM_TID == 0) scal[3] -= 0.5 * xrx;
      DFM_SYNC();
      const double ll = scal[3];
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
        double v = in_frozen ? Ppinf[i * R + j] : GPS(t)[i * R + j];
        a.PsF[(size_t)b * T * NP + e] = v;
      }
    }
    if (DFM_TID == 0) { a.iters[b] = it > a.max_iter ? a.max_iter : it; a.status[b] = status; }
#ifndef DFM_EMU
    if (a.done) __threadfence_system();            // results visible to the copy engine before the host is told
#endif
    DFM_SYNC();
#ifndef DFM_EMU
    if (a.done && threadIdx.x == 0) *(volatile int*)(a.done + b) = 1;
#endif
  }
}

#undef SCRP
#undef GSC
#undef GPS
// ================================================================================================
// Fused ALS kernel: the reference's least-squares "EM" (estimate_factor!, dfm_functions.ipynb:352-370)
// for BALANCED panels without constraints, one CTA per panel, all sweeps in one launch, on the same
// TMA ring + DMMA passes as k_em_fused2:
//   Lambda-step (:355-362):  Lam = (X'F)(F'F)^-1        = M pass + r x r inverse
//   F-step      (:364-365):  F   = (X Lam)(Lam'Lam)^-1  = E pass (unit weights) + r x r inverse
//   SSR         (:366):      sum x^2 - sum_t b_t'(Lam'Lam)^-1 b_t,  b_t = Lam'x_t   (no third pass)
//   stop        (:367-368):  |dSSR| < tol T N
// Panels with missing data / constraints / odd T use the general kernels (k_als_lambda, k_als_factor).
struct AlsFusedArgs {
  const double* Xs;     // [B][N][T] standardised, no NaN
  double* F;            // [B][T*r] column-major: in = starting factors, out = final factors
  double* Lam;          // [B][N*r] column-major out
  AlsState* st;         // tss / nobs already set; ssr, iters, done, status written here
  int B, T, N;
  double tol;
  long long max_iter;
  int l2_win[2];        // turn window per panel pass (copies): full rounds, tail round (f2_round_win)
};

template <int R>
__global__ void DFM_FUSED2_BOUNDS k_als_fused2(AlsFusedArgs a, const DFM_GRID_CONSTANT CUtensorMap tmap) {
  DFM_SMEM(sm);
  constexpr int RR = R * R;
  const int T = a.T, N = a.N;
  const int Tp = pad4mod16(T), Np = pad4mod16(N);
  double* Z = sm;                          // [FZ][Tp]
  double* Lam = Z + (size_t)FZ * Tp;       // [R][Np]
  double* FtF = Lam + (size_t)R * Np;  double* Gi = FtF + RR;  double* LtL = Gi + RR;  double* Hi = LtL + RR;
  double* tmp = Hi + RR;                   // 2R
  double* red = tmp + 2 * R;               // 40
  int* ctl = (int*)(red + 40);             // [0] = bad, [1] = turn window of the panel (f2_produce)
  double* part = red + 48;                 // 2 * F2_NCW * 72
  double* ring = part + 2 * F2_NCW * 72;
#ifndef DFM_EMU
  ring += ((128u - (f2_smem_u32(ring) & 127u)) & 127u) / 8;
  __shared__ uint64_t fullb[F2_S], emptyb[F2_S];
  if (threadIdx.x == 0) { for (int s_ = 0; s_ < F2_S; ++s_) { f2_mbar_init(&fullb[s_], 1); f2_mbar_init(&emptyb[s_], F2_NCW); } }
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  __syncthreads();
  F2Ring rg; rg.ring = ring; rg.full = fullb; rg.empty = emptyb; rg.rs = 0; rg.rph = 0; rg.wrap = false;
  const long long nitems = (long long)((N + 8 * F2_SBS - 1) / (8 * F2_SBS)) * ((T + F2_TC - 1) / F2_TC);
#endif
  for (int b = DFM_BX; b < a.B; b += DFM_GX) {
#ifdef DFM_EMU
    const double* X = a.Xs + (size_t)b * T * N;
#endif
    for (int e = DFM_TID; e < FZ * Tp; e += DFM_NT) Z[e] = 0.0;
    DFM_SYNC();
    for (int e = DFM_TID; e < T * R; e += DFM_NT) { int t = e % T, c = e / T; Z[ZI(t, c)] = a.F[(size_t)b * T * R + e]; }
    if (DFM_TID == 0) ctl[0] = 0;
#ifndef DFM_EMU
    if (DFM_TID == 0) ctl[1] = f2_round_win(a.l2_win, a.B, b);
#endif
    DFM_SYNC();
    double ssr = 0.0, ssr_old = 0.0, tss = 0.0;              // tss = sum x^2 of the panel, summed in the first F-step
    long long it = 0;
    int status = 0;
    while (it < a.max_iter) {
      // ---------------- Lambda-step
      for (int e = DFM_TID; e < RR; e += DFM_NT) {
        int i = e / R, j = e % R; double s = 0.0;
        for (int t = 0; t < T; ++t) s += Z[ZI(t, i)] * Z[ZI(t, j)];
        FtF[e] = s;
      }
      DFM_SYNC();
      if (DFM_WARP == 0) w_inv<R>(Gi, FtF, tmp, &ctl[0]);
#ifdef DFM_EMU
      for (int n = 0; n < N; ++n) {
        double acc[R];
        for (int c = 0; c < R; ++c) acc[c] = 0.0;
        for (int t = 0; t < T; ++t) { double x = X[(size_t)n * T + t]; for (int c = 0; c < R; ++c) acc[c] += x * Z[ZI(t, c)]; }
        for (int c = 0; c < R; ++c) Lam[LI(n, c)] = acc[c];
      }
#else
      // (no sum of squares here: the first F-step sums it)
      if (DFM_WARP == 0) f2_produce(rg, &tmap, b * N, T, N, /*c_outer=*/false, &ctl[1]);
      else if (DFM_WARP <= F2_NCW) f2_consume_M<R, false>(rg, DFM_WARP - 1, T, N, Tp, Np, Z, Lam, nullptr, part);
      else rg.skip(nitems);
#endif
      DFM_SYNC();
      for (int n = DFM_TID; n < N; n += DFM_NT) {             // Lam_n = (F'F)^-1 S_xf,n
        double sx[R], lam[R];
#pragma unroll
        for (int c = 0; c < R; ++c) sx[c] = Lam[LI(n, c)];
#pragma unroll
        for (int i = 0; i < R; ++i) { double s = 0.0;
#pragma unroll
          for (int j = 0; j < R; ++j) s += Gi[i * R + j] * sx[j]; lam[i] = s; }
#pragma unroll
        for (int c = 0; c < R; ++c) Lam[LI(n, c)] = lam[c];
      }
      DFM_SYNC();
      // ---------------- F-step
      for (int e = DFM_TID; e < RR; e += DFM_NT) {
        int i = e / R, j = e % R; double s = 0.0;
        for (int n = 0; n < N; ++n) s += Lam[LI(n, i)] * Lam[LI(n, j)];
        LtL[e] = s;
      }
      DFM_SYNC();
      if (DFM_WARP == 0) w_inv<R>(Hi, LtL, tmp, &ctl[0]);
      double tssp = 0.0;
#ifdef DFM_EMU
      for (int t = 0; t < T; ++t) {
        for (int c = 0; c < FZ; ++c) Z[ZI(t, c)] = 0.0;
        for (int n = 0; n < N; ++n) { double x = X[(size_t)n * T + t]; if (it == 0) tssp += x * x; for (int c = 0; c < R; ++c) Z[ZI(t, c)] += x * Lam[LI(n, c)]; }
      }
#else
      if (DFM_WARP == 0) f2_produce(rg, &tmap, b * N, T, N, /*c_outer=*/true, &ctl[1]);
      else if (DFM_WARP <= F2_NCW) {
        if (it == 0) tssp = f2_consume_E<R, true>(rg, DFM_WARP - 1, T, N, Tp, Np, Z, Lam);
        else f2_consume_E<R, false>(rg, DFM_WARP - 1, T, N, Tp, Np, Z, Lam);
      } else rg.skip(nitems);
#endif
      DFM_SYNC();
      double bf = 0.0;
      for (int t = DFM_TID; t < T; t += DFM_NT) {              // f_t = (Lam'Lam)^-1 b_t ; b_t'f_t
        double bb[R], f[R];
#pragma unroll
        for (int j = 0; j < R; ++j) bb[j] = Z[ZI(t, j)];
#pragma unroll
        for (int i = 0; i < R; ++i) { double s = 0.0;
#pragma unroll
          for (int j = 0; j < R; ++j) s += Hi[i * R + j] * bb[j]; f[i] = s; bf += s * bb[i]; }
#pragma unroll
        for (int i = 0; i < R; ++i) Z[ZI(t, i)] = f[i];
      }
      bf = block_sum(bf, red);
      if (it == 0) tss = block_sum(tssp, red);
      ssr_old = ssr; ssr = tss - bf;
      ++it;
      if (ctl[0]) { status = 3; break; }
      if (!(fabs(ssr_old - ssr) >= a.tol * (double)T * (double)N)) break;            // :367-368
      if (it >= a.max_iter) { status = 4; break; }
    }
    for (int e = DFM_TID; e < T * R; e += DFM_NT) { int t = e % T, c = e / T; a.F[(size_t)b * T * R + e] = Z[ZI(t, c)]; }
    for (int e = DFM_TID; e < N * R; e += DFM_NT) { int i = e % N, c = e / N; a.Lam[(size_t)b * N * R + e] = Lam[LI(i, c)]; }
    if (DFM_TID == 0) { a.st[b].ssr_old = ssr_old; a.st[b].ssr = ssr; a.st[b].iters = (int)it; a.st[b].done = 1; a.st[b].status = status; }
    DFM_SYNC();
  }
}

template <int R>
inline size_t als_fused2_smem_doubles(int T, int N) {
  return (size_t)FZ * pad4mod16(T) + (size_t)R * pad4mod16(N) + 4 * (size_t)R * R + 2 * R + 48 +
         2 * F2_NCW * 72 + (size_t)F2_S * F2_STG + 26;
}

template <int R>
inline size_t fused2_smem_doubles(int T, int N) {
  return (size_t)FZ * pad4mod16(T) + (size_t)R * pad4mod16(N) + 3 * (size_t)N + 30 * (size_t)R * R + 2 * R + 40 + 8 + 8 +
         std::max((size_t)97 * R + (size_t)R * R, (size_t)2 * F2_NCW * 72) + (size_t)F2_S * F2_STG + 26;
}

}  // namespace dfm
