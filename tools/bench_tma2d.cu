// bench_tma2d.cu -- microbenchmark of the panel-streaming ring used by k_em_fused2 / k_als_fused2:
// one 2-D tensor-map TMA per stage (box = bc periods x br series), mbarrier full/empty ring, consumer
// warps doing a few FP64 DMMAs per stage.  Sweeps box shape, ring depth, producer count, consumer
// work and CTAs per SM to find what bounds the pass (issue rate, latency x bytes in flight, DRAM).
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -o tools/bench_tma2d.bin tools/bench_tma2d.cu
#include <cuda.h>
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <vector>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %d\n", cudaGetErrorString(e), __LINE__); exit(1); } } while (0)

struct P { int B, T, N, bc, br, S, nprod, ncons, work; };

__device__ __forceinline__ uint32_t s32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mb_init(uint64_t* b, int n) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(s32(b)), "r"(n)); }
__device__ __forceinline__ void mb_expect(uint64_t* b, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(s32(b)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mb_arrive(uint64_t* b) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(s32(b)) : "memory"); }
__device__ __forceinline__ void mb_wait(uint64_t* b, uint32_t ph) {
  uint32_t ok;
  do {
    asm volatile("{\n.reg .pred p;\nmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\nselp.u32 %0, 1, 0, p;\n}" : "=r"(ok) : "r"(s32(b)), "r"(ph) : "memory");
  } while (!ok);
}
__device__ __forceinline__ void tma2d(void* dst, const CUtensorMap* tm, int c0, int c1, uint64_t* bar) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
               ::"r"(s32(dst)), "l"(tm), "r"(c0), "r"(c1), "r"(s32(bar)) : "memory");
}

__global__ void __launch_bounds__(256) k_ring(const __grid_constant__ CUtensorMap tm, P p, double* out) {
  extern __shared__ __align__(128) unsigned char smraw[];
  double* ring = (double*)(((uintptr_t)smraw + 127) & ~(uintptr_t)127);
  const int stage = p.br * p.bc;
  uint64_t* full = (uint64_t*)(ring + (size_t)p.S * stage);
  uint64_t* empty = full + p.S;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int s = 0; s < p.S; ++s) { mb_init(&full[s], 1); mb_init(&empty[s], p.ncons); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const int nck = (p.T + p.bc - 1) / p.bc, nsb = (p.N + p.br - 1) / p.br;
  const int per_panel = nck * nsb;
  int npan = 0;
  for (int b = blockIdx.x; b < p.B; b += gridDim.x) ++npan;
  const long long total = (long long)npan * per_panel;
  double acc0 = 0.0, acc1 = 0.0;
  // ring position tracked incrementally (no integer divisions on the critical path)
  if (warp < p.nprod) {
    int slot = warp % p.S, turn = warp / p.S;
    int pi = 0, r = warp;                       // panel index of this CTA, item within the panel
    while (r >= per_panel) { r -= per_panel; ++pi; }
    for (long long it = warp; it < total; it += p.nprod) {
      if (turn > 0) mb_wait(&empty[slot], (uint32_t)((turn - 1) & 1));
      if (lane == 0) {
        const int b = blockIdx.x + pi * gridDim.x, c = r / nsb, sb = r - c * nsb;
        mb_expect(&full[slot], (uint32_t)(stage * 8));
        tma2d(ring + (size_t)slot * stage, &tm, c * p.bc, b * p.N + sb * p.br, &full[slot]);
      }
      __syncwarp();
      slot += p.nprod; while (slot >= p.S) { slot -= p.S; ++turn; }
      r += p.nprod; while (r >= per_panel) { r -= per_panel; ++pi; }
    }
  } else if (warp < p.nprod + p.ncons) {
    int slot = 0; uint32_t ph = 0;
    for (long long it = 0; it < total; ++it) {
      mb_wait(&full[slot], ph);
      const double* tile = ring + (size_t)slot * stage;
      for (int k = 0; k < p.work; k += 2) {
        double a0 = tile[((lane & 3) + (k & 4)) * p.bc + (lane >> 2) + 8 * (warp - p.nprod)];
        double a1 = tile[((lane & 3) + (k & 4)) * p.bc + (lane >> 2) + 8 * (warp - p.nprod) + 48];
        double d0 = acc0, d1 = acc1, e0 = acc1, e1 = acc0;
        asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n" : "+d"(d0), "+d"(d1) : "d"(a0), "d"(a1));
        asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n" : "+d"(e0), "+d"(e1) : "d"(a1), "d"(a0));
        acc0 = d0 + e1; acc1 = d1 + e0;
      }
      if (p.work == 0) acc0 += tile[lane];
      __syncwarp();
      if (lane == 0) mb_arrive(&empty[slot]);
      if (++slot == p.S) { slot = 0; ph ^= 1; }
    }
  }
  if (acc0 + acc1 == 123.456) out[blockIdx.x] = acc0;
}


// K tensor copies issued back to back by one thread into K slots with K mbarriers, then waited for:
// cycles(K) ~ cycles(1) means the copies overlap, ~ K * cycles(1) means they are serialised.
__global__ void __launch_bounds__(32) k_lat(const __grid_constant__ CUtensorMap tm, int bc, int br, int K, int reps, int rows_total, long long* out, int bulk1d,
                                            const double* X, int T) {
  extern __shared__ __align__(128) unsigned char smraw[];
  double* ring = (double*)(((uintptr_t)smraw + 127) & ~(uintptr_t)127);
  const int stage = bc * br;
  uint64_t* bars = (uint64_t*)(ring + (size_t)K * stage);
  if (threadIdx.x == 0) {
    for (int k = 0; k < K; ++k) mb_init(&bars[k], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    long long tot = 0, mn = 1ll << 60;
    for (int r = 0; r < reps; ++r) {
      long long t0 = clock64();
      for (int k = 0; k < K; ++k) {
        int row = (int)(((long long)blockIdx.x * reps * K + (long long)r * K + k) * br % (rows_total - br));
        mb_expect(&bars[k], (uint32_t)(stage * 8));
        if (!bulk1d) tma2d(ring + (size_t)k * stage, &tm, 0, row, &bars[k]);
        else asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                          ::"r"(s32(ring + (size_t)k * stage)), "l"(X + (size_t)row * T), "r"(stage * 8), "r"(s32(&bars[k])) : "memory");
      }
      long long t1 = clock64();
      for (int k = 0; k < K; ++k) mb_wait(&bars[k], (uint32_t)(r & 1));
      long long t2 = clock64();
      tot += t2 - t0; if (t2 - t0 < mn) mn = t2 - t0;
      if (r == reps - 1) out[blockIdx.x * 4 + 2] = t1 - t0;
    }
    out[blockIdx.x * 4] = tot / reps; out[blockIdx.x * 4 + 1] = mn;
  }
}

typedef CUresult (*encode_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                              const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

int main(int argc, char** argv) {
  int nsm = 0; CK(cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, 0));
  const int B = 8 * nsm, T = 500, N = 200;   // no tail at any of the grids used
  double* X; double* out;
  size_t n = (size_t)B * N * T;
  CK(cudaMalloc(&X, n * 8)); CK(cudaMalloc(&out, 4096 * 8));
  CK(cudaMemset(X, 0, n * 8));
  void* fp = nullptr; cudaDriverEntryPointQueryResult q;
  CK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fp, cudaEnableDefault, &q));
  encode_fn enc = (encode_fn)fp;
  CK(cudaFuncSetAttribute(k_ring, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
  cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));

  {  // ---- overlap test
    long long* lo; CK(cudaMalloc(&lo, nsm * 4 * 8));
    std::vector<long long> h(nsm * 4);
    CK(cudaFuncSetAttribute(k_lat, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    printf("overlap test: cycles for K copies issued back to back by one thread (avg / min / issue-only), grid CTAs of 32 threads\n");
    struct LC { int bc, br, grid, bulk; };
    for (LC lc : {LC{100, 8, 1, 0}, LC{100, 8, nsm, 0}, LC{16, 50, 1, 0}, LC{16, 50, nsm, 0}, LC{100, 8, 1, 1}, LC{100, 8, nsm, 1}, LC{250, 8, nsm, 0}}) {
      CUtensorMap tm;
      cuuint64_t dims[2] = {(cuuint64_t)T, (cuuint64_t)B * N}; cuuint64_t strides[1] = {(cuuint64_t)T * 8};
      cuuint32_t box[2] = {(cuuint32_t)lc.bc, (cuuint32_t)lc.br}, es[2] = {1, 1};
      CUresult rc = enc(&tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT64, 2, X, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                        CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
      if (rc != CUDA_SUCCESS) { printf("encode failed\n"); continue; }
      for (int K : {1, 2, 4, 8}) {
        size_t smem = (size_t)K * lc.bc * lc.br * 8 + K * 8 + 256;
        k_lat<<<lc.grid, 32, smem>>>(tm, lc.bc, lc.br, K, 20, B * N, lo, lc.bulk, X, T);
        CK(cudaDeviceSynchronize());
        CK(cudaMemcpy(h.data(), lo, lc.grid * 4 * 8, cudaMemcpyDeviceToHost));
        double a = 0, m = 0, is = 0; for (int g = 0; g < lc.grid; ++g) { a += h[g * 4]; m += h[g * 4 + 1]; is += h[g * 4 + 2]; }
        printf("  %s box %3dx%-3d grid %3d K=%d : avg %7.0f  min %7.0f  issue %6.0f cyc\n", lc.bulk ? "bulk1d" : "tensor", lc.bc, lc.br, lc.grid, K, a / lc.grid, m / lc.grid, is / lc.grid);
      }
    }
  }
  struct Cfg { int bc, br, S, nprod, ncons, work, grid; };
  std::vector<Cfg> cfgs;
  for (int grid : {nsm, 2 * nsm}) {
    cfgs.push_back({100, 8, 6, 1, 6, 4, grid});     // the shipped configuration
    cfgs.push_back({100, 8, 6, 1, 6, 0, grid});     // no consumer math
    cfgs.push_back({100, 8, 6, 2, 6, 4, grid});     // two producer warps
    cfgs.push_back({100, 8, 4, 1, 6, 4, grid});     // shallower / deeper rings
    cfgs.push_back({100, 8, 8, 1, 6, 4, grid});
    cfgs.push_back({100, 8, 12, 1, 6, 4, grid});
    cfgs.push_back({100, 16, 3, 1, 6, 8, grid});    // taller boxes
    cfgs.push_back({100, 16, 4, 1, 6, 8, grid});
    cfgs.push_back({100, 16, 6, 1, 6, 8, grid});
    cfgs.push_back({100, 40, 2, 1, 6, 8, grid});
    cfgs.push_back({128, 8, 6, 1, 6, 4, grid});     // wider boxes (4 chunks of 128 cover T = 500)
    cfgs.push_back({250, 8, 3, 1, 6, 8, grid});
    cfgs.push_back({250, 8, 4, 1, 6, 8, grid});
    cfgs.push_back({252, 8, 5, 1, 6, 8, grid});
  }
  cfgs.push_back({100, 8, 6, 1, 6, 4, nsm / 2});    // half the SMs, one CTA each: is the cap per CTA or chip-wide?
  cfgs.push_back({100, 8, 12, 1, 6, 4, nsm / 2});
  cfgs.push_back({100, 16, 6, 1, 6, 8, nsm / 2});
  printf("%-5s %-4s %-3s %-5s %-5s %-5s %-5s %10s %10s %12s\n", "bc", "br", "S", "nprod", "ncons", "work", "grid", "ms", "GB/s", "cyc/stage");
  for (auto& c : cfgs) {
    CUtensorMap tm;
    cuuint64_t dims[2] = {(cuuint64_t)T, (cuuint64_t)B * N}; cuuint64_t strides[1] = {(cuuint64_t)T * 8};
    cuuint32_t box[2] = {(cuuint32_t)c.bc, (cuuint32_t)c.br}, es[2] = {1, 1};
    CUresult rc = enc(&tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT64, 2, X, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                      CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (rc != CUDA_SUCCESS) { printf("encode failed %d for bc=%d br=%d\n", (int)rc, c.bc, c.br); continue; }
    P p{B, T, N, c.bc, c.br, c.S, c.nprod, c.ncons, c.work};
    size_t smem = (size_t)c.S * c.bc * c.br * 8 + 2 * c.S * 8 + 256;
    // force the intended residency: pad shared memory so that exactly one (grid <= SM count) or two CTAs fit per SM
    size_t pad = (c.grid > nsm) ? 100 * 1024 : 120 * 1024;
    if (smem < pad) smem = pad;
    for (int w = 0; w < 2; ++w) k_ring<<<c.grid, 256, smem>>>(tm, p, out);
    CK(cudaDeviceSynchronize());
    CK(cudaEventRecord(e0));
    const int reps = 3;
    for (int w = 0; w < reps; ++w) k_ring<<<c.grid, 256, smem>>>(tm, p, out);
    CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1));
    float ms; CK(cudaEventElapsedTime(&ms, e0, e1)); ms /= reps;
    CK(cudaGetLastError());
    const int nck = (T + c.bc - 1) / c.bc, nsb = (N + c.br - 1) / c.br;
    double stages_per_cta = (double)B / c.grid * nck * nsb;
    double cyc = ms * 1e-3 * 1.9e9 / stages_per_cta;
    printf("%-5d %-4d %-3d %-5d %-5d %-5d %-5d %10.3f %10.1f %12.0f\n", c.bc, c.br, c.S, c.nprod, c.ncons, c.work, c.grid, ms, n * 8.0 / ms / 1e6, cyc);
  }
  return 0;
}
