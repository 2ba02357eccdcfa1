// bench_stream.cu -- dev micro-benchmark (not product): what HBM rate do the fused kernel's two panel
// passes reach at its occupancy (128 threads, ~71 KB smem => 3 CTAs/SM), for several load schemes?
// build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/bench_stream.bin tools/bench_stream.cu
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>
#include <cstdint>

#define T 500
#define N 200
#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %d\n", cudaGetErrorString(e), __LINE__); exit(1); } } while (0)

__device__ __forceinline__ void dmma(double& d0, double& d1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n" : "+d"(d0), "+d"(d1) : "d"(a), "d"(b));
}
__device__ __forceinline__ double ld_pf256(const double* p) {
  double v; asm volatile("ld.global.nc.L2::256B.f64 %0, [%1];" : "=d"(v) : "l"(p)); return v;
}

// ---- E pattern (column-major X, tile 8 t x 4 series): U loads in flight
template <int U, bool PF>
__global__ void __launch_bounds__(128, 3) k_e(const double* __restrict__ Xall, int B, double* out) {
  extern __shared__ double sm[];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, lr = lane >> 2, lc = lane & 3;
  double acc = 0;
  for (int b = blockIdx.x; b < B; b += gridDim.x) {
    const double* X = Xall + (size_t)b * T * N;
    for (int rb = w; rb < (T + 7) / 8; rb += 4) {
      int t = rb * 8 + lr; bool tok = t < T; const double* xp = X + (tok ? t : 0);
      double d0 = 0, d1 = 0;
      for (int i0 = 0; i0 < N; i0 += 4 * U) {
        double av[U];
#pragma unroll
        for (int u = 0; u < U; ++u) { int n = i0 + 4 * u + lc; av[u] = (tok && n < N) ? (PF ? ld_pf256(xp + (size_t)n * T) : __ldg(xp + (size_t)n * T)) : 0.0; }
#pragma unroll
        for (int u = 0; u < U; ++u) if (i0 + 4 * u < N) dmma(d0, d1, av[u], sm[(i0 + 4 * u + lc) * 8 + lr]);
      }
      acc += d0 + d1;
    }
  }
  if (acc == 1.2345) out[0] = acc;
}

// ---- M pattern (column-major X, tile 8 series x 4 t)
template <int U>
__global__ void __launch_bounds__(128, 3) k_m(const double* __restrict__ Xall, int B, double* out) {
  extern __shared__ double sm[];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, lr = lane >> 2, lc = lane & 3;
  double acc = 0;
  for (int b = blockIdx.x; b < B; b += gridDim.x) {
    const double* X = Xall + (size_t)b * T * N;
    for (int sb = w; sb < N / 8; sb += 4) {
      const double* xp = X + (size_t)(sb * 8 + lr) * T;
      double d0 = 0, d1 = 0;
      for (int t0 = 0; t0 < T; t0 += 4 * U) {
        double av[U];
#pragma unroll
        for (int u = 0; u < U; ++u) { int t = t0 + 4 * u + lc; av[u] = (t < T) ? __ldg(xp + t) : 0.0; }
#pragma unroll
        for (int u = 0; u < U; ++u) if (t0 + 4 * u < T) dmma(d0, d1, av[u], sm[((t0 + 4 * u + lc) % 500) * 8 + lr]);
      }
      acc += d0 + d1;
    }
  }
  if (acc == 1.2345) out[0] = acc;
}

// ---- M pattern with 16-byte loads: tile 8 series x 8 t per 2 DMMAs (k-index permutation)
template <int U>
__global__ void __launch_bounds__(128, 3) k_m16(const double* __restrict__ Xall, int B, double* out) {
  extern __shared__ double sm[];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, lr = lane >> 2, lc = lane & 3;
  double acc = 0;
  for (int b = blockIdx.x; b < B; b += gridDim.x) {
    const double* X = Xall + (size_t)b * T * N;
    for (int sb = w; sb < N / 8; sb += 4) {
      const double2* xp = reinterpret_cast<const double2*>(X + (size_t)(sb * 8 + lr) * T);
      double d0 = 0, d1 = 0;
      for (int t0 = 0; t0 < T; t0 += 8 * U) {
        double2 av[U];
#pragma unroll
        for (int u = 0; u < U; ++u) { int t = t0 + 8 * u + 2 * lc; av[u] = (t < T) ? __ldg(xp + t / 2) : make_double2(0, 0); }
#pragma unroll
        for (int u = 0; u < U; ++u) if (t0 + 8 * u < T) {
          int t = t0 + 8 * u + 2 * lc;
          dmma(d0, d1, av[u].x, sm[(t % 500) * 8 + lr]); dmma(d0, d1, av[u].y, sm[((t + 1) % 500) * 8 + lr]);
        }
      }
      acc += d0 + d1;
    }
  }
  if (acc == 1.2345) out[0] = acc;
}

// ---- plain coalesced read (16 B per lane, 512 B per warp instruction), same occupancy
template <int U>
__global__ void __launch_bounds__(128, 3) k_copy(const double* __restrict__ Xall, int B, double* out) {
  extern __shared__ double sm[];
  double acc = 0;
  for (int b = blockIdx.x; b < B; b += gridDim.x) {
    const double2* X = reinterpret_cast<const double2*>(Xall + (size_t)b * T * N);
    for (int i = threadIdx.x; i < T * N / 2; i += 128 * U) {
      double2 v[U];
#pragma unroll
      for (int u = 0; u < U; ++u) v[u] = (i + 128 * u < T * N / 2) ? __ldg(X + i + 128 * u) : make_double2(0, 0);
#pragma unroll
      for (int u = 0; u < U; ++u) acc += v[u].x + v[u].y;
    }
  }
  if (acc == 1.2345) out[0] = acc + sm[0];
}

// ---- TMA 1D bulk copies into a shared-memory ring (M pattern: a stage = 8 series x TC periods)
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, int cnt) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(cnt)); }
__device__ __forceinline__ void mbar_expect(uint64_t* bar, uint32_t bytes) { asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory"); }
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory"); }
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t phase) {
  asm volatile("{\n.reg .pred p;\nWAIT_%=:\nmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n@p bra DONE_%=;\nbra WAIT_%=;\nDONE_%=:\n}" ::"r"(smem_u32(bar)), "r"(phase) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
#define TC 100           // periods per stage: 8 series x 100 x 8 B = 6.4 KB
#define TS 100           // smem row stride (doubles); 100 % 16 = 4 -> conflict-free fragments
template <int S>
__global__ void __launch_bounds__(128, 3) k_m_tma(const double* __restrict__ Xall, int B, double* out) {
  extern __shared__ __align__(128) double sm[];
  double* ring = sm;                               // S stages x 8 x TS
  double* zb = sm + S * 8 * TS;                    // fake B operand
  __shared__ uint64_t full[S], empty[S];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, lr = lane >> 2, lc = lane & 3;
  if (threadIdx.x == 0) { for (int s = 0; s < S; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 3); } }
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  __syncthreads();
  // work items: (panel, series block sb 0..24, t-chunk c 0..4); consumers = warps 1..3, producer = warp 0 lane 0
  const int per_panel = (N / 8) * (T / TC);
  long long nitems = 0;
  for (int b = blockIdx.x; b < B; b += gridDim.x) nitems += per_panel;
  double acc = 0;
  if (w == 0) {
    if (lane == 0) {
      long long it = 0;
      for (int b = blockIdx.x; b < B; b += gridDim.x) {
        const double* X = Xall + (size_t)b * T * N;
        for (int item = 0; item < per_panel; ++item, ++it) {
          int s = it % S; uint32_t ph = (it / S) & 1;
          if (it >= S) mbar_wait(&empty[s], ph ^ 1);
          int sb = item / (T / TC), c = item % (T / TC);
          mbar_expect(&full[s], 8 * TC * 8);
          for (int r = 0; r < 8; ++r) bulk_g2s(ring + (size_t)s * 8 * TS + r * TS, X + (size_t)(sb * 8 + r) * T + c * TC, TC * 8, &full[s]);
        }
      }
    }
  } else {
    double d0 = 0, d1 = 0;
    for (long long it = 0; it < nitems; ++it) {
      int s = it % S; uint32_t ph = (it / S) & 1;
      mbar_wait(&full[s], ph);
      const double* tile = ring + (size_t)s * 8 * TS;
      // the 3 consumer warps split the TC/4 k-chunks of the stage
      for (int kc = w - 1; kc < TC / 4; kc += 3) dmma(d0, d1, tile[lr * TS + kc * 4 + lc], zb[(kc * 4 + lc) * 8 + lr]);
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[s]);
    }
    acc = d0 + d1;
  }
  if (acc == 1.2345) out[0] = acc;
}


// ---- producer-issue experiment: 256 threads; the 8 row copies of a stage are issued by
//   MODE 0: lane 0 of warp 0 (serial)   MODE 1: lanes 0..7 of warp 0   MODE 2: lane 0 of warps 0..NPW-1 (rows strided)
template <int S, int MODE, int NPW>
__global__ void __launch_bounds__(256, 2) k_m_tma2(const double* __restrict__ Xall, int B, double* out) {
  extern __shared__ __align__(128) double sm[];
  double* ring = sm; double* zb = sm + S * 8 * TS;
  __shared__ uint64_t full[S], empty[S];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, lr = lane >> 2, lc = lane & 3;
  constexpr int NPROD = (MODE == 2) ? NPW : 1;
  constexpr int NCONS = 8 - NPROD;
  if (threadIdx.x == 0) { for (int s = 0; s < S; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], NCONS); } }
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  __syncthreads();
  const int per_panel = (N / 8) * (T / TC);
  long long nitems = 0;
  for (int b = blockIdx.x; b < B; b += gridDim.x) nitems += per_panel;
  double acc = 0;
  if (w < NPROD) {
    long long it = 0;
    for (int b = blockIdx.x; b < B; b += gridDim.x) {
      const double* X = Xall + (size_t)b * T * N;
      for (int item = 0; item < per_panel; ++item, ++it) {
        int s = it % S; uint32_t ph = (it / S) & 1;
        if (it >= S) mbar_wait(&empty[s], ph ^ 1);
        int sb = item / (T / TC), c = item % (T / TC);
        if (w == 0 && lane == 0) mbar_expect(&full[s], 8 * TC * 8);
        __syncwarp();
        if (MODE == 0) { if (lane == 0) for (int r = 0; r < 8; ++r) bulk_g2s(ring + (size_t)s * 8 * TS + r * TS, X + (size_t)(sb * 8 + r) * T + c * TC, TC * 8, &full[s]); }
        else if (MODE == 1) { if (lane < 8) bulk_g2s(ring + (size_t)s * 8 * TS + lane * TS, X + (size_t)(sb * 8 + lane) * T + c * TC, TC * 8, &full[s]); }
        else { if (lane == 0) for (int r = w; r < 8; r += NPROD) bulk_g2s(ring + (size_t)s * 8 * TS + r * TS, X + (size_t)(sb * 8 + r) * T + c * TC, TC * 8, &full[s]); }
      }
    }
  } else {
    const int cw = w - NPROD;
    double d0 = 0, d1 = 0, e0 = 0, e1 = 0;
    for (long long it = 0; it < nitems; ++it) {
      int s = it % S; uint32_t ph = (it / S) & 1;
      mbar_wait(&full[s], ph);
      const double* tile = ring + (size_t)s * 8 * TS;
      for (int kc = cw; kc < TC / 4; kc += 2 * NCONS) {
        dmma(d0, d1, tile[lr * TS + kc * 4 + lc], zb[(kc * 4 + lc) * 8 + lr]);
        if (kc + NCONS < TC / 4) dmma(e0, e1, tile[lr * TS + (kc + NCONS) * 4 + lc], zb[((kc + NCONS) * 4 + lc) * 8 + lr]);
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[s]);
    }
    acc = d0 + d1 + e0 + e1;
  }
  if (acc == 1.2345) out[0] = acc;
}

template <typename F>
void run(const char* name, F launch, double bytes) {
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  launch(); CK(cudaDeviceSynchronize());
  cudaEventRecord(e0); for (int i = 0; i < 5; ++i) launch(); cudaEventRecord(e1); CK(cudaDeviceSynchronize());
  float ms; cudaEventElapsedTime(&ms, e0, e1); ms /= 5;
  printf("%-34s %8.3f ms  %8.1f GB/s\n", name, ms, bytes / ms / 1e6);
}

int main() {
  const int B = 1250;
  size_t n = (size_t)B * T * N;
  double* X; double* out; CK(cudaMalloc(&X, n * 8)); CK(cudaMalloc(&out, 64)); CK(cudaMemset(X, 0, n * 8));
  const int smem = 71 * 1024; const int grid = 444;
  double bytes = (double)n * 8;
#define SET(k) CK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, smem))
  SET((k_e<10, false>)); SET((k_e<25, false>)); SET((k_e<10, true>)); SET((k_e<25, true>)); SET(k_m<10>); SET(k_m<25>); SET(k_m16<8>); SET(k_m16<16>);
  SET(k_copy<4>); SET(k_copy<8>); SET(k_m_tma<4>); SET(k_m_tma<8>);
  run("E ldg8 U=10", [&] { k_e<10, false><<<grid, 128, smem>>>(X, B, out); }, bytes);
  run("E ldg8 U=25", [&] { k_e<25, false><<<grid, 128, smem>>>(X, B, out); }, bytes);
  run("E ldg8 U=10 L2::256B", [&] { k_e<10, true><<<grid, 128, smem>>>(X, B, out); }, bytes);
  run("E ldg8 U=25 L2::256B", [&] { k_e<25, true><<<grid, 128, smem>>>(X, B, out); }, bytes);
  run("M ldg8 U=10", [&] { k_m<10><<<grid, 128, smem>>>(X, B, out); }, bytes);
  run("M ldg8 U=25", [&] { k_m<25><<<grid, 128, smem>>>(X, B, out); }, bytes);
  run("M ldg16 U=8", [&] { k_m16<8><<<grid, 128, smem>>>(X, B, out); }, bytes);
  run("M ldg16 U=16", [&] { k_m16<16><<<grid, 128, smem>>>(X, B, out); }, bytes);
  run("copy 16B U=4", [&] { k_copy<4><<<grid, 128, smem>>>(X, B, out); }, bytes);
  run("copy 16B U=8", [&] { k_copy<8><<<grid, 128, smem>>>(X, B, out); }, bytes);
  run("M TMA bulk ring S=4 (6.4KB/stage)", [&] { k_m_tma<4><<<grid, 128, smem>>>(X, B, out); }, bytes);
  run("M TMA bulk ring S=8", [&] { k_m_tma<8><<<grid, 128, smem>>>(X, B, out); }, bytes);
  // occupancy 2 CTAs/SM variants (grid 296) to see the sensitivity
  run("E ldg8 U=25 grid296", [&] { k_e<25, false><<<296, 128, smem>>>(X, B, out); }, bytes);
  run("M TMA S=8 grid296", [&] { k_m_tma<8><<<296, 128, smem>>>(X, B, out); }, bytes);
  run("copy 16B U=8 grid296", [&] { k_copy<8><<<296, 128, smem>>>(X, B, out); }, bytes);
  {
    const int smem2 = 110 * 1024;
#define SET2(k) CK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, smem2))
    SET2((k_m_tma2<5, 0, 1>)); SET2((k_m_tma2<5, 1, 1>)); SET2((k_m_tma2<5, 2, 2>)); SET2((k_m_tma2<5, 2, 4>)); SET2((k_m_tma2<10, 1, 1>)); SET2((k_m_tma2<10, 2, 4>));
    run("256thr 2/SM S=5  1 lane x 8 copies", [&] { k_m_tma2<5, 0, 1><<<296, 256, smem2>>>(X, B, out); }, bytes);
    run("256thr 2/SM S=5  8 lanes of one warp", [&] { k_m_tma2<5, 1, 1><<<296, 256, smem2>>>(X, B, out); }, bytes);
    run("256thr 2/SM S=5  lane0 of 2 warps", [&] { k_m_tma2<5, 2, 2><<<296, 256, smem2>>>(X, B, out); }, bytes);
    run("256thr 2/SM S=5  lane0 of 4 warps", [&] { k_m_tma2<5, 2, 4><<<296, 256, smem2>>>(X, B, out); }, bytes);
    run("256thr 2/SM S=10 8 lanes of one warp", [&] { k_m_tma2<10, 1, 1><<<296, 256, smem2>>>(X, B, out); }, bytes);
    run("256thr 2/SM S=10 lane0 of 4 warps", [&] { k_m_tma2<10, 2, 4><<<296, 256, smem2>>>(X, B, out); }, bytes);
  }
  return 0;
}
