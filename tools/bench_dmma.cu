// bench_dmma.cu -- FP64 tensor-core MMA issue rate on sm_90a by shape (m8n8k4 / m16n8k4 / m16n8k8 / m16n8k16)
// and plain DFMA, with 1..4 warps per SM sub-partition, independent accumulators.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -o tools/bench_dmma.bin tools/bench_dmma.cu
#include <cuda_runtime.h>
#include <cstdio>
#include <vector>
#include <cstdlib>
#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %d\n", cudaGetErrorString(e), __LINE__); exit(1); } } while (0)

template <int SHAPE, int NACC>
__global__ void k(int iters, double* out, long long* cyc) {
  double a0 = threadIdx.x * 1e-3, a1 = a0 + 1, a2 = a0 + 2, a3 = a0 + 3, a4 = a0 + 4, a5 = a0 + 5, a6 = a0 + 6, a7 = a0 + 7;
  double b0 = 1.0 + threadIdx.x * 1e-6, b1 = b0 + 1e-3, b2 = b0 + 2e-3, b3 = b0 + 3e-3;
  double d[NACC][4];
#pragma unroll
  for (int j = 0; j < NACC; ++j) { d[j][0] = j; d[j][1] = j + 1; d[j][2] = j + 2; d[j][3] = j + 3; }
  __syncthreads();
  long long t0 = clock64();
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int j = 0; j < NACC; ++j) {
      if (SHAPE == 0)
        asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(d[j][0]), "+d"(d[j][1]) : "d"(a0), "d"(b0));
      else if (SHAPE == 1)
        asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};"
                     : "+d"(d[j][0]), "+d"(d[j][1]), "+d"(d[j][2]), "+d"(d[j][3]) : "d"(a0), "d"(a1), "d"(b0));
      else if (SHAPE == 2)
        asm volatile("mma.sync.aligned.m16n8k8.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                     : "+d"(d[j][0]), "+d"(d[j][1]), "+d"(d[j][2]), "+d"(d[j][3]) : "d"(a0), "d"(a1), "d"(a2), "d"(a3), "d"(b0), "d"(b1));
      else if (SHAPE == 3)
        asm volatile("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, {%12,%13,%14,%15}, {%0,%1,%2,%3};"
                     : "+d"(d[j][0]), "+d"(d[j][1]), "+d"(d[j][2]), "+d"(d[j][3])
                     : "d"(a0), "d"(a1), "d"(a2), "d"(a3), "d"(a4), "d"(a5), "d"(a6), "d"(a7), "d"(b0), "d"(b1), "d"(b2), "d"(b3));
      else if (SHAPE == 4) { d[j][0] = fma(a0, b0, d[j][0]); d[j][1] = fma(a1, b1, d[j][1]); d[j][2] = fma(a2, b2, d[j][2]); d[j][3] = fma(a3, b3, d[j][3]); }
      else if (SHAPE == 5) { d[j][0] = fma(a0, b0, d[j][0]); }                       // one dependent DFMA chain
      else if (SHAPE == 6) { d[j][0] = d[j][0] + a0; }                               // one dependent DADD chain
      else if (SHAPE == 7) { d[j][0] = __shfl_sync(0xffffffffu, d[j][0], (threadIdx.x + 1) & 7, 8); }   // 64-bit shuffle chain
      else if (SHAPE == 8) { d[j][0] = d[j][0] * b0; }                               // DMUL chain
    }
  }
  long long t1 = clock64();
  double s = 0;
#pragma unroll
  for (int j = 0; j < NACC; ++j) s += d[j][0] + d[j][1] + d[j][2] + d[j][3];
  if (s == 123.456) out[0] = s;
  if (threadIdx.x == 0) cyc[blockIdx.x] = t1 - t0;
}

template <int SHAPE, int NACC>
void run(const char* name, double fma_per_op, int warps) {
  int nsm = 0; CK(cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, 0));
  double* out; long long* cyc; CK(cudaMalloc(&out, 8)); CK(cudaMalloc(&cyc, nsm * 8));
  const int iters = 2000;
  k<SHAPE, NACC><<<nsm, warps * 32>>>(iters, out, cyc); CK(cudaDeviceSynchronize());
  k<SHAPE, NACC><<<nsm, warps * 32>>>(iters, out, cyc); CK(cudaDeviceSynchronize());
  std::vector<long long> h(nsm); CK(cudaMemcpy(h.data(), cyc, nsm * 8, cudaMemcpyDeviceToHost));
  double c = 0; for (int i = 0; i < nsm; ++i) c += h[i]; c /= nsm;
  double ops_per_warp = (double)iters * NACC;
  double per_smsp = c / (ops_per_warp * warps / 4.0);          // cycles per op per sub-partition (warps spread over 4 SMSPs)
  double fma_clk_sm = ops_per_warp * warps * fma_per_op / c;
  int khz = 0; CK(cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, 0));
  printf("%-22s acc=%d warps/SM=%2d : %7.1f cyc/op/warp  %6.1f cyc/op/SMSP  %6.1f FMA/clk/SM  (%.1f TFLOP/s at %.2f GHz x %d SMs)\n", name, NACC,
         warps, c / ops_per_warp, per_smsp, fma_clk_sm, fma_clk_sm * 2 * nsm * khz * 1e3 / 1e12, khz * 1e-6, nsm);
  cudaFree(out); cudaFree(cyc);
}

int main() {
  run<5, 1>("DFMA dependent chain", 32, 4); run<6, 1>("DADD dependent chain", 32, 4); run<8, 1>("DMUL dependent chain", 32, 4);
  run<7, 1>("SHFL.64 dependent chain", 32, 4); run<5, 1>("DFMA dep chain, 16 warps", 32, 16);
  for (int w : {4, 8, 16}) {
    if (w == 4) { run<0, 1>("DMMA m8n8k4 (dep chain)", 256, 4); run<3, 1>("DMMA m16n8k16 (dep chain)", 2048, 4); }
    if (w == 4) { run<0, 8>("DMMA m8n8k4", 256, 4); run<1, 8>("DMMA m16n8k4", 512, 4); run<2, 8>("DMMA m16n8k8", 1024, 4); run<3, 8>("DMMA m16n8k16", 2048, 4); run<4, 8>("DFMA x4 per lane", 128, 4); }
    if (w == 8) { run<0, 8>("DMMA m8n8k4", 256, 8); run<1, 8>("DMMA m16n8k4", 512, 8); run<2, 8>("DMMA m16n8k8", 1024, 8); run<3, 8>("DMMA m16n8k16", 2048, 8); run<4, 8>("DFMA x4 per lane", 128, 8); }
    if (w == 16) { run<0, 8>("DMMA m8n8k4", 256, 16); run<1, 8>("DMMA m16n8k4", 512, 16); run<2, 8>("DMMA m16n8k8", 1024, 16); run<3, 8>("DMMA m16n8k16", 2048, 16); run<4, 8>("DFMA x4 per lane", 128, 16); }
  }
  return 0;
}
