// dfm_api.cu -- the C-ABI (include/dfm_b200.h): handle, workspace, H2D/D2H staging and the launch
// sequences of every entry point.  Host code here only orchestrates; all arithmetic runs in the
// kernels.  There is no CPU compute path: without a CUDA device dfm_create fails.
#include "../../include/dfm_b200.h"
#include "dfm_common.cuh"
#include "dfm_kernels_np.cuh"
#include "dfm_kernels_em.cuh"
#include "dfm_kernels_emb.cuh"
#include "dfm_kernels_ss.cuh"
#include "dfm_kernels_fused.cuh"
#include "dfm_kernels_fused2.cuh"
#include "dfm_kernels_als_masked.cuh"
#include "dfm_kernels_rep.cuh"
#include "dfm_kernels_inst.cuh"
#include "dfm_kernels_sim.cuh"
#include "dfm_kernels_news.cuh"
#include <algorithm>
#include <new>
#include <thread>
#include <type_traits>
#include <vector>
#ifndef DFM_EMU
#include <dlfcn.h>
#else
#include <map>
#include <mutex>
#endif

#ifdef DFM_EMU
// ---- minimal CUDA-runtime stand-ins for the host-emulation test build -------------------------
typedef int cudaError_t;
enum { cudaSuccess = 0, cudaErrorInvalidValue = 1, cudaErrorInvalidConfiguration = 9 };
// The launch limits of the H100 that the emulated launches are held to, so that a launch the device would refuse fails
// here too: it does not run, and the next cudaGetLastError() returns the error (the entry point then returns DFM_ERR_CUDA).
static thread_local cudaError_t g_emu_last_err = cudaSuccess;
static std::mutex g_emu_attr_mu;
static std::map<const void*, size_t> g_emu_smem_attr;        // cudaFuncAttributeMaxDynamicSharedMemorySize per kernel
static inline void emu_set_error(cudaError_t e) { if (g_emu_last_err == cudaSuccess) g_emu_last_err = e; }
static inline void emu_set_smem(const void* kern, size_t bytes) {
  if (bytes > 227 * 1024) { emu_set_error(cudaErrorInvalidValue); return; }   // the attribute's ceiling on sm_90
  std::lock_guard<std::mutex> lk(g_emu_attr_mu);
  g_emu_smem_attr[kern] = bytes;
}
static inline bool emu_launch_ok(const void* kern, long long gx, long long gy, long long nt, size_t smem) {
  size_t attr = 0;
  {
    std::lock_guard<std::mutex> lk(g_emu_attr_mu);
    auto it = g_emu_smem_attr.find(kern);
    if (it != g_emu_smem_attr.end()) attr = it->second;
  }
  const bool ok = smem <= std::max<size_t>(48 * 1024, attr) && nt >= 1 && nt <= 1024 && gx >= 1 && gx <= 2147483647LL && gy >= 1 &&
                  gy <= 65535;
  if (!ok) emu_set_error(cudaErrorInvalidConfiguration);
  return ok;
}
enum cudaMemcpyKind { cudaMemcpyHostToDevice, cudaMemcpyDeviceToHost, cudaMemcpyDeviceToDevice };
static inline cudaError_t cudaMalloc(void** p, size_t n) { *p = malloc(n ? n : 1); return *p ? 0 : 2; }
static inline cudaError_t cudaFree(void* p) { free(p); return 0; }
static inline cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, cudaMemcpyKind, cudaStream_t) { memcpy(d, s, n); return 0; }
static inline cudaError_t cudaMemsetAsync(void* d, int v, size_t n, cudaStream_t) { memset(d, v, n); return 0; }
static inline cudaError_t cudaMemcpy2DAsync(void* d, size_t dp, const void* s, size_t sp, size_t w, size_t rows, cudaMemcpyKind, cudaStream_t) {
  for (size_t j = 0; j < rows; ++j) memcpy((char*)d + j * dp, (const char*)s + j * sp, w);
  return 0;
}
static inline cudaError_t cudaStreamCreate(cudaStream_t* s) { *s = nullptr; return 0; }
static inline cudaError_t cudaStreamDestroy(cudaStream_t) { return 0; }
static inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return 0; }
static inline cudaError_t cudaSetDevice(int) { return 0; }
static inline cudaError_t cudaGetDeviceCount(int* n) { *n = 1; return 0; }
static inline cudaError_t cudaGetLastError() { cudaError_t e = g_emu_last_err; g_emu_last_err = cudaSuccess; return e; }
static inline const char* cudaGetErrorString(cudaError_t e) {
  return e == cudaErrorInvalidConfiguration ? "emu: launch past a device limit (grid, block or shared memory)"
       : e == cudaErrorInvalidValue ? "emu: shared-memory attribute past the device limit" : "emu";
}
#define DFM_SET_SMEM(kern, bytes) emu_set_smem((const void*)(kern), (size_t)(bytes))    // (kern: a kernel or a pointer to one)
#else
#define DFM_SET_SMEM(kern, bytes) cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(bytes))
#endif

using namespace dfm;

struct ProfRec { const char* name; 
#ifndef DFM_EMU
  cudaEvent_t e0, e1;
#endif
};

struct dfm_handle {
  int device;
  int nsm;                     // streaming multiprocessors of the device: sizes grids and the per-panel CTA plans
  int l2_bytes;                // L2 cache size: sizes the share of each resident panel the TMA kernels keep in L2
  cudaStream_t stream;
  cudaStream_t copy_stream;    // second stream: the H2D copies of the streaming host path run here, under the EM kernel
  cudaStream_t d2h_stream;     // third stream: results of finished panels go back while the kernel is still running
  int* done_host; int* done_dev; size_t done_cap;   // per-panel completion flags (mapped pinned memory, written by the kernel)
  int* pinned_one;             // pinned host int == 1: source of the stream-ordered "chunk has landed" flag copies
  bool own_stream;
  char* ws;
  size_t ws_bytes;
  long long launches;
  int profile;                 // 1: bracket every kernel launch with CUDA events (dfm_profile_*)
  std::vector<ProfRec>* prof;
  char err[256];
};

namespace {

const size_t kMaxSmem = 220 * 1024;
const int kMaxReadyChunks = 4096;
// Entry points whose launches put the batch on gridDim.y (at most 65535 blocks) refuse larger batches with
// DFM_ERR_UNSUPPORTED; callers split such batches.
const int kMaxGridBatch = 65535;

struct Arena {
  char* base; size_t off;
  explicit Arena(char* b) : base(b), off(0) {}
  template <typename Tp> Tp* get(size_t n) {
    size_t bytes = (n * sizeof(Tp) + 255) & ~(size_t)255;
    Tp* p = base ? reinterpret_cast<Tp*>(base + off) : nullptr;
    off += bytes;
    return p;
  }
};

int fail(dfm_handle* h, int code, const char* msg) {
  if (h) { snprintf(h->err, sizeof(h->err), "%s", msg); }
  return code;
}

#define CK(call)                                                                                   \
  do { cudaError_t e__ = (call); if (e__ != cudaSuccess) {                                         \
    snprintf(h->err, sizeof(h->err), "%s:%d %s", __FILE__, __LINE__, cudaGetErrorString(e__));    \
    return DFM_ERR_CUDA; } } while (0)

#ifdef DFM_EMU
#define PROF_BEGIN(name) ((void)0)
#define PROF_END() ((void)0)
#else
#define PROF_BEGIN(name_)                                                                          \
  ProfRec pr__; pr__.name = name_;                                                                 \
  if (h->profile) { cudaEventCreate(&pr__.e0); cudaEventCreate(&pr__.e1); cudaEventRecord(pr__.e0, h->stream); }
#define PROF_END() if (h->profile) { cudaEventRecord(pr__.e1, h->stream); h->prof->push_back(pr__); }
#endif
#ifdef DFM_EMU
#define L(kern, gx, gy, nt, smem, ...)                                                             \
  do { if (emu_launch_ok((const void*)(kern), (gx), (gy), (nt), (smem))) DFM_LAUNCH(kern, gx, gy, nt, smem, h->stream, __VA_ARGS__); \
       h->launches++; } while (0)
#else
#define L(kern, gx, gy, nt, smem, ...)                                                             \
  do { PROF_BEGIN(#kern); DFM_LAUNCH(kern, gx, gy, nt, smem, h->stream, __VA_ARGS__); PROF_END(); h->launches++; } while (0)
#endif

int ensure_ws(dfm_handle* h, size_t bytes) {
  if (bytes <= h->ws_bytes) return DFM_OK;
  if (h->ws) { CK(cudaStreamSynchronize(h->stream)); CK(cudaFree(h->ws)); h->ws = nullptr; h->ws_bytes = 0; }
  size_t want = bytes + (bytes >> 3) + (1 << 20);
  void* p = nullptr;
  CK(cudaMalloc(&p, want));
  h->ws = (char*)p; h->ws_bytes = want;
  return DFM_OK;
}

// input staging: returns device pointer for `src` (copying if it lives on the host)
template <typename Tp>
int stage_in(dfm_handle* h, const Tp* src, Tp* dev_buf, size_t n, int mem, const Tp** out) {
  if (mem == DFM_MEM_DEVICE) { *out = src; return DFM_OK; }
  CK(cudaMemcpyAsync(dev_buf, src, n * sizeof(Tp), cudaMemcpyHostToDevice, h->stream));
  *out = dev_buf;
  return DFM_OK;
}
template <typename Tp>
int copy_out(dfm_handle* h, Tp* dst, const Tp* dev, size_t n, int mem) {
  if (!dst || dst == dev) return DFM_OK;
  CK(cudaMemcpyAsync(dst, dev, n * sizeof(Tp), mem == DFM_MEM_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, h->stream));
  return DFM_OK;
}

int finish(dfm_handle* h, int mem) {
  CK(cudaGetLastError());
  if (mem == DFM_MEM_HOST) CK(cudaStreamSynchronize(h->stream));
  return DFM_OK;
}

// threads per block for the thread-per-period kernels: ws doubles of shared memory per thread
int tpt_threads(int ws_doubles) {
  int nt = (int)((96 * 1024) / ((size_t)ws_doubles * 8));
  nt = (nt / 32) * 32;
  return std::max(32, std::min(128, nt));
}

}  // namespace

// any NaN in the panel / parameters?  (the fused path handles balanced panels only)
namespace dfm {
__global__ void k_em_scan_fused(const double* __restrict__ X, const double* __restrict__ Lam, const double* __restrict__ R,
                                int T, int N, int r, int* flag) {
  int i = DFM_BX, b = DFM_BY;
  const double* x = X + ((size_t)b * N + i) * T;
  int bad = 0;
  for (int t = DFM_TID; t < T; t += DFM_NT) if (is_nan(x[t])) bad = 1;
  if (DFM_TID == 0) { for (int a = 0; a < r; ++a) if (is_nan(Lam[(size_t)b * N * r + i + (size_t)N * a])) bad = 1; if (is_nan(R[(size_t)b * N + i])) bad = 1; }
  if (bad) *flag = 1;
}
}  // namespace dfm

// [T, rows] FP64 view of a batch of column-major panels with the fused kernels' F2_TS x 8 box
static int make_panel_tmap(dfm_handle* h, const double* X, int T, long long rows, CUtensorMap* out) {
#ifdef DFM_EMU
  (void)h; (void)X; (void)T; (void)rows; memset(out, 0, sizeof(*out));
  return DFM_OK;
#else
  typedef CUresult (*encode_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
  static encode_fn fn = nullptr;
  if (!fn) {
    void* p = nullptr; cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || !p)
      return fail(h, DFM_ERR_CUDA, "cuTensorMapEncodeTiled not available");
    fn = (encode_fn)p;
  }
  cuuint64_t dims[2] = {(cuuint64_t)T, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)T * 8};
  cuuint32_t box[2] = {F2_TS, 8 * F2_SBS}, es[2] = {1, 1};
  CUresult rc = fn(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT64, 2, (void*)X, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (rc != CUDA_SUCCESS) { snprintf(h->err, sizeof(h->err), "cuTensorMapEncodeTiled failed (%d)", (int)rc); return DFM_ERR_CUDA; }
  return DFM_OK;
#endif
}

// f(std::integral_constant<int, V>{}) for the run-time value v = V in [Lo, Hi]: the one place where a run-time size
// (r for the fused kernels, the column-block count for the contraction kernels) picks a kernel template.  The
// callers have checked the range; a value outside it takes Hi.
template <int Lo, int Hi, typename F>
static auto dispatch(int v, F&& f) {
  if constexpr (Lo == Hi) return f(std::integral_constant<int, Lo>{});
  else {
    if (v == Lo) return f(std::integral_constant<int, Lo>{});
    return dispatch<Lo + 1, Hi>(v, f);
  }
}

// Grid of a persistent kernel that loops over the B panels: as many CTAs as are resident on the device at once.  The
// fused kernels' scratch has one row per CTA for min(B, nsm * 8) CTAs, which bounds the emulation build's grid too.
template <typename K>
static int resident_grid(const dfm_handle* h, K kern, int threads, size_t smem, int B) {
#ifdef DFM_EMU
  (void)threads;
  DFM_SET_SMEM(kern, smem);
  return std::min(B, h->nsm * 8);
#else
  DFM_SET_SMEM(kern, smem);
  int occ = 1;
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, threads, smem);
  if (occ < 1) occ = 1;
  return std::min(B, h->nsm * occ);
#endif
}

// Series-block groups per panel that `grid` CTAs of a TMA kernel keep in L2 at evict-last priority (f2_keep_stages):
// F2_L2KEEP_PCT of L2 split over the CTAs active in a round; keep[0] for the full rounds, keep[1] for the tail round.
static void l2_keep_plan(const dfm_handle* h, int grid, int B, int T, int N, int keep[2]) {
  const long long budget = (long long)h->l2_bytes * F2_L2KEEP_PCT / 100, group = 64LL * F2_SBS * T;   // 64 T bytes per 8 series
  const long long nsg = (N + 8 * F2_SBS - 1) / (8 * F2_SBS);
  const int tail = (B % grid) ? B % grid : grid;
  keep[0] = (int)std::min(nsg, budget / (grid * group));
  keep[1] = (int)std::min(nsg, budget / (tail * group));
}

// One launch of the fused EM kernel over all panels of fa (fa.scratch: min(B, nsm * 8) * T * FUSED_SCR(r) doubles):
// k_em_fused2 (TMA panel ring, even T) when use2, else k_em_fused.
static int launch_em_fused(dfm_handle* h, FusedArgs fa, int r, bool use2) {
  return dispatch<1, 8>(r, [&](auto R) -> int {
    constexpr int RT = decltype(R)::value;
    if (use2) {
      const size_t smem = fused2_smem_doubles<RT>(fa.T, fa.N) * 8;
      const int grid = resident_grid(h, k_em_fused2<RT>, 256, smem, fa.B);
      l2_keep_plan(h, grid, fa.B, fa.T, fa.N, fa.l2_keep);
      CUtensorMap tm; int rc = make_panel_tmap(h, fa.X, fa.T, (long long)fa.B * fa.N, &tm); if (rc) return rc;
      L(k_em_fused2<RT>, grid, 1, 256, smem, fa, tm);
    } else {
      const size_t smem = fused_smem_doubles<RT>(fa.T, fa.N) * 8;
      const int grid = resident_grid(h, k_em_fused<RT>, 128, smem, fa.B);
      L(k_em_fused<RT>, grid, 1, 128, smem, fa);
    }
    return DFM_OK;
  });
}

// Multi-CTA contraction kernels of the general path for balanced panels (dfm_kernels_emb.cuh): split factors and buffers.
struct EmbPlan {
  bool on; int ncb, ntE, nsE, nper, ntM, tsM, tper;
  double *Bpart, *qpart, *Spart, *sxxpart, *Cpart; int* counters;
  size_t smE, smM;
};
static EmbPlan emb_plan(int T, int N, int r, int batch, int nsm) {
  EmbPlan e{};
  e.on = r <= 32;
  if (!e.on) return e;
  e.ncb = (r + 7) / 8;
  const int target = 2 * nsm;
  e.ntE = (T + EMB_TILE - 1) / EMB_TILE;
  int want = (target + e.ntE * batch - 1) / (e.ntE * batch);
  int ns = std::max((N + EMB_MAXSPLIT - 1) / EMB_MAXSPLIT, std::min(want, (N + 31) / 32));
  e.nper = (((N + ns - 1) / ns) + 3) & ~3;
  e.nsE = (N + e.nper - 1) / e.nper;
  e.ntM = (N + EMB_TILE - 1) / EMB_TILE;
  want = (target + e.ntM * batch - 1) / (e.ntM * batch);
  int ts = std::max(1, std::min(want, (T + 31) / 32));
  e.tper = (((T + ts - 1) / ts) + 3) & ~3;
  e.tsM = (T + e.tper - 1) / e.tper;
  if ((long long)e.nsE * batch > 65535 || (long long)e.tsM * batch > 65535) { e.on = false; return e; }
  e.smE = ((size_t)e.ncb * 8 * emb_pad(e.nper) + e.nper + 48) * 8;
  e.smM = ((size_t)2 * r * r + (size_t)2 * EMB_TILE * (r + 1) + 96) * 8;
  return e;
}
static void emb_launch_E(dfm_handle* h, const EmbPlan& e, const double* x, const double* dW, const double* dR, const double* dlogR, int T, int N,
                         int r, int batch, double* dBt, double* dqt, double* dslr, int* dnt, EmState* st) {
  dispatch<1, 4>(e.ncb, [&](auto C) {
    constexpr int NCB = decltype(C)::value;
    DFM_SET_SMEM(k_emb_contract<NCB>, e.smE);
    L(k_emb_contract<NCB>, e.ntE, e.nsE * batch, 256, e.smE, x, dW, dR, dlogR, T, N, r, e.nsE, e.nper, batch, e.Bpart, e.qpart, e.counters,
      dBt, dqt, dslr, dnt, st);
  });
}
static void emb_launch_M(dfm_handle* h, const EmbPlan& e, const double* x, const double* dFs, const double* dSff, int T, int N, int r, int batch,
                         double* dL, double* dR, double* dW, double* dlogR, EmState* st) {
  dispatch<1, 4>(e.ncb, [&](auto C) {
    constexpr int NCB = decltype(C)::value;
    DFM_SET_SMEM(k_emb_mstep<NCB>, e.smM);
    L(k_emb_mstep<NCB>, e.ntM, e.tsM * batch, 256, e.smM, x, dFs, dSff, T, N, r, e.tsM, e.tper, batch, e.Spart, e.sxxpart,
      e.counters + (size_t)batch * e.ntE, dL, dR, dW, dlogR, e.Cpart, st);
  });
}

// Device scratch of the general EM path for B panels of T periods.  dfm_em_kalman and dfm_kalman_smooth (on the panels
// padded to T + H periods) allocate it with gen_bufs; the multi-CTA contraction partials only when emb.on.
struct GenBufs {
  double *An, *Qn, *W, *logR, *C, *Bt, *qt, *slr;
  int* nt;                                        // [2][B][T]: n_t, then src_t of the frozen-step logic
  double *Ct, *zp, *zf, *Pp, *Pf, *Sff;
  double* xch;                                    // cluster exchange (scalars, boundary states, Gram partials)
  EmbPlan emb;
};
static GenBufs gen_bufs(Arena& a, const EmbPlan& emb, size_t B, int T, int N, int r, int p) {
  const size_t k = (size_t)r * p, kk = k * k, rr = (size_t)r * r, rk = r * k, np = (size_t)r * (r + 1) / 2;
  GenBufs g;
  g.An = a.get<double>(B * rk); g.Qn = a.get<double>(B * rr); g.W = a.get<double>(B * N * r); g.logR = a.get<double>(B * N);
  g.C = a.get<double>(B * rr); g.Bt = a.get<double>(B * T * r); g.qt = a.get<double>(B * T); g.slr = a.get<double>(B * T);
  g.nt = a.get<int>(2 * B * T); g.Ct = a.get<double>(B * T * np); g.zp = a.get<double>(B * T * k); g.zf = a.get<double>(B * T * k);
  g.Pp = a.get<double>(B * T * kk); g.Pf = a.get<double>(B * T * kk); g.Sff = a.get<double>(B * rr);
  g.xch = a.get<double>(B * (16 + 64 * k + 16 * (kk + rk)));
  g.emb = emb;
  if (emb.on) {
    g.emb.Bpart = a.get<double>((size_t)emb.nsE * B * T * r); g.emb.qpart = a.get<double>((size_t)emb.nsE * B * T);
    g.emb.Spart = a.get<double>((size_t)emb.tsM * B * N * r); g.emb.sxxpart = a.get<double>((size_t)emb.tsM * B * N);
    g.emb.Cpart = a.get<double>(B * emb.ntM * rr); g.emb.counters = a.get<int>(B * (size_t)(emb.ntE + emb.ntM));
  }
  return g;
}

// Device buffers of one dfm_em_kalman call that its fused and general paths share: the uploaded panels (host input
// only), the parameters updated in place, the results, and the fused kernels' scratch.
struct EmBufs {
  double *X, *L, *R, *A, *Q, *P0, *Fs, *PsF, *ll, *PF;
  EmState* st;
  int *it, *stat, *active, *flag;
  int* ready;                                     // streaming host path: one "landed" flag per chunk of panels
  double* scratch;                                // fused kernels: min(B, nsm * 8) * T * FUSED_SCR(r) doubles
};
static FusedArgs fused_args(const EmBufs& d, const dfm_em_opts* o, const double* x) {
  FusedArgs fa{};
  fa.X = x; fa.Lam = d.L; fa.R = d.R; fa.A = d.A; fa.Q = d.Q; fa.P0 = d.P0; fa.Fs = d.Fs; fa.PsF = d.PsF; fa.loglik = d.ll;
  fa.iters = d.it; fa.status = d.stat; fa.scratch = d.scratch; fa.B = o->batch; fa.T = o->T; fa.N = o->N; fa.max_iter = o->max_iter;
  fa.tol = o->tol;
  return fa;
}

// Staging tile (periods) of the frozen-run phases of k_em_filter_smooth: few panels -> large tiles (one CTA per SM
// anyway); many panels -> the largest tile that still lets two CTAs share an SM, if any does.
static int fs_stage_periods(int nsm, int batch, int r, int p) {
  int stgT = (batch <= nsm) ? 256 : 16;
  const size_t lim2 = 112 * 1024;
  if (batch <= nsm) { while (stgT > 8 && em_fs_smem_doubles(r, p, stgT) * 8 > kMaxSmem) stgT /= 2; }
  else if (em_fs_smem_doubles(r, p, 4) * 8 <= lim2) { while (stgT > 4 && em_fs_smem_doubles(r, p, stgT) * 8 > lim2) stgT /= 2; }
  else { while (stgT > 4 && em_fs_smem_doubles(r, p, stgT) * 8 > kMaxSmem) stgT /= 2; }
  return stgT;
}

// CTAs per panel (thread-block cluster) of the filter / smoother
static int fs_cluster_size(const dfm_handle* h, int batch, const double* dxch) {
  int ncl = 1;
  if (dxch) { if (batch * 8 <= h->nsm) ncl = 8; else if (batch * 4 <= h->nsm) ncl = 4; else if (batch * 2 <= h->nsm) ncl = 2; }
  if (getenv("DFM_CLUSTER")) ncl = std::max(1, std::min(8, atoi(getenv("DFM_CLUSTER"))));
  return ncl;
}

// One launch of k_em_filter_smooth over the batch (T periods in g); a cluster per panel when ncl > 1 (set to 1 if the
// cluster cannot be placed).  A, Q, mi, tol and want_psf are the caller's: the EM loop's, or one E-step at fixed parameters.
static int launch_filter_smooth(dfm_handle* h, int& ncl, const GenBufs& g, int batch, int T, int r, int p, const double* dA, const double* dQ,
                                const double* dP0, double* dFs, double* dPsF, double* dll, EmState* st, int mi, double tol, int want_psf) {
  const int stgT = fs_stage_periods(h->nsm, batch, r, p);
  const size_t smFS = em_fs_smem_doubles(r, p, stgT) * 8;
  const int ntFS = (batch <= 2 * h->nsm) ? 512 : 256;     // few panels: more warps for the parallel frozen runs; many: two CTAs per SM
  int* dsrc = g.nt + (size_t)batch * T;
#ifndef DFM_EMU
  if (ncl > 1) {
    // few panels: a thread-block cluster per panel (the CTAs split the parallel phases of the frozen runs)
    PROF_BEGIN("k_em_filter_smooth");
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)(batch * ncl)); cfg.blockDim = dim3((unsigned)ntFS); cfg.dynamicSmemBytes = smFS; cfg.stream = h->stream;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeClusterDimension; at[0].val.clusterDim.x = (unsigned)ncl; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
    cfg.attrs = at; cfg.numAttrs = 1;
    cudaError_t ce = cudaLaunchKernelEx(&cfg, k_em_filter_smooth, dA, dQ, dP0, g.C, g.Bt, g.qt, g.slr, g.nt, g.Ct, T, r, p, g.zp, g.zf,
                                        g.Pp, g.Pf, dFs, dPsF, g.Sff, g.An, g.Qn, dll, mi, tol, st, dsrc, stgT, want_psf, g.xch);
    PROF_END(); h->launches++;
    if (ce == cudaSuccess) return DFM_OK;
    (void)cudaGetLastError();                      // the cluster could not be placed: run the plain one-CTA-per-panel launch instead
    ncl = 1;
  }
#endif
  L(k_em_filter_smooth, batch, 1, ntFS, smFS, dA, dQ, dP0, g.C, g.Bt, g.qt, g.slr, g.nt, g.Ct, T, r, p, g.zp, g.zf, g.Pp, g.Pf,
    dFs, dPsF, g.Sff, g.An, g.Qn, dll, mi, tol, st, dsrc, stgT, want_psf, (double*)nullptr);
  return DFM_OK;
}

// General multi-kernel EM path on device-resident data (any r, p, missing data).
static int run_em_general(dfm_handle* h, const double* x, const dfm_em_opts* o, const EmBufs& d, const GenBufs& g, int want_psf) {
  const int T = o->T, N = o->N, r = o->r, p = o->p, batch = o->batch, mi = o->max_iter;
  const int np = r * (r + 1) / 2;
  const int ntC = tpt_threads(np + r), nblkC = (T + ntC - 1) / ntC;
  const EmbPlan& emb = g.emb;
  int ncl = fs_cluster_size(h, batch, g.xch);
  L(k_em_state_init, batch, 1, 1, 0, d.st);
  L(k_em_scan, N, batch, 64, 0, x, d.L, T, N, r, d.st);
  L(k_em_prep, batch, 1, 128, 0, d.L, d.R, N, r, p, g.W, g.logR, g.C, d.A, g.An, d.Q, g.Qn, d.st, mi, 0, emb.on ? 1 : 0);
  if (emb.on) {
    L(k_emb_cinit, emb.ntM, batch, 256, 0, d.L, g.W, N, r, emb.Cpart, d.st);
    L(k_emb_close, batch, 1, 256, 0, N, r, p, emb.ntM, emb.Cpart, g.C, d.A, g.An, d.Q, g.Qn, d.st, mi, 0);
  }
  // how many panels have missing data?  (decides which contraction kernels are launched at all: one sync, before the loop)
  int n_missing = batch;
  if (emb.on) {
    L(k_em_count_missing, 1, 1, 128, 48 * 8, d.st, batch, d.active);
    CK(cudaMemcpyAsync(&n_missing, d.active, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    CK(cudaMemsetAsync(emb.counters, 0, sizeof(int) * (size_t)batch * (emb.ntE + emb.ntM), h->stream));
  }
  const bool any_missing = n_missing > 0, any_bal = emb.on ? (n_missing < batch) : true;
  const int emb_on = emb.on ? 1 : 0;
  int h_active = batch;
  for (int it = 0; it < mi && h_active > 0; ++it) {
    if (any_missing) L(k_em_contract, nblkC, batch, ntC, ((size_t)(np + r) * ntC + 8) * 8, x, d.L, g.W, d.R, g.logR, g.C, T, N, r, g.Bt, g.qt, g.slr, g.nt, g.Ct, d.st);
    if (any_bal) {                                                          // (each returns at once for panels of the other kind)
      if (!emb.on) L(k_em_contract_bal, (T + 31) / 32, batch, 256, 8 * 32 * 3 * 8, x, g.W, d.R, g.logR, T, N, r, g.Bt, g.qt, g.slr, g.nt, d.st);
      else emb_launch_E(h, emb, x, g.W, d.R, g.logR, T, N, r, batch, g.Bt, g.qt, g.slr, g.nt, d.st);
    }
    launch_filter_smooth(h, ncl, g, batch, T, r, p, d.A, d.Q, d.P0, d.Fs, d.PsF, d.ll, d.st, mi, o->tol, want_psf);
    if (any_missing || !emb.on) L(k_em_mstep_series, N, batch, 64, (size_t)(2 * np + r + 8) * 8, x, d.Fs, d.PsF, g.Sff, T, N, r, d.L, d.R, d.st, emb_on);
    if (any_bal && emb.on) {
      emb_launch_M(h, emb, x, d.Fs, g.Sff, T, N, r, batch, d.L, d.R, g.W, g.logR, d.st);
      L(k_emb_close, batch, 1, 256, 0, N, r, p, emb.ntM, emb.Cpart, g.C, d.A, g.An, d.Q, g.Qn, d.st, mi, 1);
    }
    if (any_missing || !emb.on) L(k_em_prep, batch, 1, 128, 0, d.L, d.R, N, r, p, g.W, g.logR, g.C, d.A, g.An, d.Q, g.Qn, d.st, mi, 1, emb_on);
    if (o->tol > 0 && ((it & 3) == 3)) {
      L(k_em_count_active, 1, 1, 128, 48 * 8, d.st, batch, d.active);
      CK(cudaMemcpyAsync(&h_active, d.active, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
      CK(cudaStreamSynchronize(h->stream));
    }
  }
  L(k_em_collect, batch, 1, 1, 0, d.st, d.it, d.stat);
  return DFM_OK;
}

static int launch_als_fused2(dfm_handle* h, AlsFusedArgs fa, int r) {
  return dispatch<1, 8>(r, [&](auto R) -> int {
    constexpr int RT = decltype(R)::value;
    const size_t smem = als_fused2_smem_doubles<RT>(fa.T, fa.N) * 8;
    const int grid = resident_grid(h, k_als_fused2<RT>, 256, smem, fa.B);
    l2_keep_plan(h, grid, fa.B, fa.T, fa.N, fa.l2_keep);
    CUtensorMap tm; int rc = make_panel_tmap(h, fa.Xs, fa.T, (long long)fa.B * fa.N, &tm); if (rc) return rc;
    L(k_als_fused2<RT>, grid, 1, 256, smem, fa, tm);
    return DFM_OK;
  });
}
static void launch_als_masked(dfm_handle* h, const AlsMaskedArgs& fa, int r) {
  dispatch<1, 8>(r, [&](auto R) {
    constexpr int RT = decltype(R)::value;
    const size_t smem = als_masked_smem_doubles<RT>(fa.T, fa.N) * 8;
    const int grid = resident_grid(h, k_als_masked<RT>, 256, smem, fa.B);
    L(k_als_masked<RT>, grid, 1, 256, smem, fa);
  });
}
static bool als_masked_shape_ok(int T, int N, int r) {
  if (r < 1 || r > 8) return false;
  return ((size_t)r * (T | 1) + (size_t)r * (N | 1) + 5 * (size_t)r * r + 48) * 8 <= 100 * 1024;
}
static bool als_fused2_shape_ok(int T, int N, int r) {
  if (r < 1 || r > 8 || T < 4 || (T & 1)) return false;
  return ((size_t)FZ * pad4mod16(T) + (size_t)r * pad4mod16(N) + (size_t)N + 4 * (size_t)r * r + 2 * r + 48 +
          2 * F2_NCW * 72 + (size_t)F2_S * F2_STG + 32) * 8 <= 113 * 1024;
}

static bool fused2_shape_ok(int T, int N, int r, int p) {
  if (p != 1 || r < 1 || r > 8 || T < 4 || (T & 1)) return false;
  size_t need = ((size_t)FZ * pad4mod16(T) + (size_t)r * pad4mod16(N) + 3 * (size_t)N + 30 * (size_t)r * r + 2 * (size_t)r +
                 std::max((size_t)97 * r + (size_t)r * r, (size_t)2 * F2_NCW * 72) + (size_t)F2_S * F2_STG + 106) * 8;
  return need <= 113 * 1024;          // two CTAs per SM
}

static bool fused_shape_ok(int T, int N, int r, int p) {
  if (p != 1 || r < 1 || r > 8 || T < 3) return false;
  return ((size_t)FZ * pad4mod16(T) + (size_t)r * pad4mod16(N) + 3 * (size_t)N + 31 * (size_t)r * r + 66 * (size_t)r + 128) * 8 <= kMaxSmem;
}

#ifndef DFM_EMU
// ---------------------------------------------------------------- streaming host path of dfm_em_kalman
// Host buffers + TMA fused kernel + more panels than are resident at once: ONE launch of the EM kernel, started
// before the data is on the device.  The copy stream uploads the batch in chunks of panels (X and the initial
// parameters), each chunk followed by a 4-byte copy that sets its "landed" flag; a CTA spins on the flag of the
// panel it is about to start (ld.acquire.sys) -- the copy engine is in order, so the flag implies the data.  The
// upload (PCIe) runs under the kernel (HBM-bound, slower than the link), P0 and the log-likelihood
// pre-fill are done inside the kernel (no other kernel can become resident next to it), and the balance check
// is deferred: a panel with NaNs ends with status 3, which triggers the scan + general-path fallback.
// (Not under a CUDA injection profiler or CUDA_LAUNCH_BLOCKING=1: launches are synchronous there, so a kernel that waits for copies
//  enqueued after its launch would never finish.  DFM_NO_PIPELINE=1 forces the upload-then-compute path too.)
static bool em_streaming_applies(const dfm_handle* h, const dfm_em_opts* o) {
  const char* clb = getenv("CUDA_LAUNCH_BLOCKING");
  const char* cdmc = getenv("CUDA_DEVICE_MAX_CONNECTIONS");
  // ... nor with CUDA_DEVICE_MAX_CONNECTIONS=1 (common in torch.distributed set-ups): all streams then share one hardware
  // queue, so the uploads could be queued BEHIND the kernel that waits for them.
  const bool profiler = getenv("CUDA_INJECTION64_PATH") || getenv("NV_COMPUTE_PROFILER_PERFWORKS_DIR") || (clb && clb[0] == '1') ||
                        (cdmc && atoi(cdmc) == 1);
  if (getenv("DFM_NO_PIPELINE") || profiler) return false;
  const int resident = dispatch<1, 8>(o->r, [&](auto R) {
    constexpr int RT = decltype(R)::value;
    return resident_grid(h, k_em_fused2<RT>, 256, fused2_smem_doubles<RT>(o->T, o->N) * 8, o->batch);
  });
  return resident < o->batch;
}

// The whole dfm_em_kalman call on the streaming host path.  Returns an error code, or DFM_OK with *fallback = false
// when the results are in `out`, or DFM_OK with *fallback = true when some panel has missing data: the panels are on
// the device then (d.X), the parameters have to be staged again, and the general path has to run on the whole batch.
static int em_streaming(dfm_handle* h, const double* X, const dfm_em_opts* o, const dfm_em_init* init, const dfm_em_out* out,
                        const EmBufs& d, bool* fallback) {
  const int T = o->T, N = o->N, r = o->r, batch = o->batch, mi = o->max_iter;
  const size_t B = batch, TN = (size_t)T * N; const int k = r * o->p, kk = k * k, rr = r * r, rk = r * k;
  *fallback = false;
  int chunk = 32;                                              // ~25 MB of C2-shaped panels: the first CTAs start early
  while ((batch + chunk - 1) / chunk > kMaxReadyChunks) chunk *= 2;
  const int nch = (batch + chunk - 1) / chunk;
  cudaStream_t cs = h->copy_stream;
  cudaEvent_t ev0 = nullptr, ev_k = nullptr;
  CK(cudaEventCreateWithFlags(&ev0, cudaEventDisableTiming));
  { cudaError_t e_ = cudaEventCreateWithFlags(&ev_k, cudaEventDisableTiming); if (e_ != cudaSuccess) { cudaEventDestroy(ev0); CK(e_); } }
#define CKE(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { cudaEventDestroy(ev0); cudaEventDestroy(ev_k); CK(e_); } } while (0)
  // the workspace is shared with whatever the previous call on this handle left in flight on h->stream (a
  // DFM_MEM_DEVICE call returns before completion): the copy stream must not touch it before that work is done
  CKE(cudaEventRecord(ev_k, h->stream));
  CKE(cudaStreamWaitEvent(cs, ev_k, 0));
  CKE(cudaStreamWaitEvent(h->d2h_stream, ev_k, 0));
  CKE(cudaMemsetAsync(d.ready, 0, (size_t)nch * sizeof(int), cs));
  CKE(cudaEventRecord(ev0, cs));
  CKE(cudaStreamWaitEvent(h->stream, ev0, 0));                   // flags are zero before the kernel can read them
  FusedArgs fa = fused_args(d, o, d.X);
  fa.ready = d.ready; fa.ready_chunk = chunk;
  if (h->done_cap < B) {                                        // completion flags the kernel writes straight into host memory
    if (h->done_host) cudaFreeHost(h->done_host);
    h->done_host = nullptr; h->done_cap = 0;
    CKE(cudaHostAlloc((void**)&h->done_host, B * sizeof(int), cudaHostAllocMapped));
    CKE(cudaHostGetDevicePointer((void**)&h->done_dev, h->done_host, 0));
    h->done_cap = B;
  }
#undef CKE
  memset(h->done_host, 0, B * sizeof(int));
  fa.done = h->done_dev;
  fa.P0out = init->P0 ? nullptr : d.P0; fa.p0_steps = 12;        // P0 in the kernel unless the caller gave one (the loglik rows are pre-filled there too)
  int rc = launch_em_fused(h, fa, r, true);
  if (rc) { cudaEventDestroy(ev0); cudaEventDestroy(ev_k); return rc; }
  cudaError_t up = cudaSuccess;                                  // first failure while enqueueing the upload
  for (int c = 0; c < nch && up == cudaSuccess; ++c) {
    size_t b0 = (size_t)c * chunk, bc = std::min<size_t>(chunk, B - b0);
#define DFM_UP(dst, src, n_) do { if (up == cudaSuccess) up = cudaMemcpyAsync((dst), (src), (size_t)(n_) * 8, cudaMemcpyHostToDevice, cs); } while (0)
    DFM_UP(d.X + b0 * TN, X + b0 * TN, bc * TN); DFM_UP(d.L + b0 * N * r, init->Lam + b0 * N * r, bc * N * r);
    DFM_UP(d.R + b0 * N, init->R + b0 * N, bc * N); DFM_UP(d.A + b0 * rk, init->A + b0 * rk, bc * rk); DFM_UP(d.Q + b0 * rr, init->Q + b0 * rr, bc * rr);
    if (init->P0) DFM_UP(d.P0 + b0 * kk, init->P0 + b0 * kk, bc * kk);
#undef DFM_UP
    if (up == cudaSuccess) up = cudaMemcpyAsync(d.ready + c, h->pinned_one, sizeof(int), cudaMemcpyHostToDevice, cs);
  }
  if (up != cudaSuccess) {
    // an upload could not be enqueued: the kernel is already running and would wait for its flags for ever ->
    // raise every flag (the CTAs then run on whatever is in the buffers), drain, report the error
    cudaMemsetAsync(d.ready, 1, (size_t)nch * sizeof(int), cs);
    cudaStreamSynchronize(cs); cudaStreamSynchronize(h->stream);
    cudaEventDestroy(ev0); cudaEventDestroy(ev_k);
    (void)cudaGetLastError();
    snprintf(h->err, sizeof(h->err), "dfm_em_kalman: host-to-device upload failed (%s)", cudaGetErrorString(up));
    return DFM_ERR_CUDA;
  }
  // results of finished panels go back on a third stream while the kernel is still running: the host polls the
  // completion flags and ships whole chunks of 128 panels in order (everything except the unpacked PF, which
  // needs a kernel of its own after the EM kernel)
  {
    const size_t dch = 128;
    volatile const int* dn = h->done_host;
    size_t next = 0; bool kernel_done = false;
    auto ship = [&](size_t b0, size_t b1) {
      const size_t nb = b1 - b0;
#define DFM_OUTS(dst, src, per) if (dst) cudaMemcpyAsync((dst) + b0 * (per), (src) + b0 * (per), nb * (per) * sizeof(*(src)), cudaMemcpyDeviceToHost, h->d2h_stream)
      DFM_OUTS(out->F, d.Fs, (size_t)T * r); DFM_OUTS(out->Lam, d.L, (size_t)N * r); DFM_OUTS(out->R, d.R, (size_t)N); DFM_OUTS(out->A, d.A, (size_t)rk);
      DFM_OUTS(out->Q, d.Q, (size_t)rr); DFM_OUTS(out->P0, d.P0, (size_t)kk); DFM_OUTS(out->loglik, d.ll, (size_t)mi);
      DFM_OUTS(out->iters, d.it, (size_t)1); DFM_OUTS(out->status, d.stat, (size_t)1);
#undef DFM_OUTS
    };
    while (next < B) {
      size_t b1 = std::min<size_t>(B, next + dch);
      bool all = true;
      if (!kernel_done) for (size_t bb = next; bb < b1; ++bb) if (!dn[bb]) { all = false; break; }
      if (all) { ship(next, b1); next = b1; continue; }
      cudaError_t q = cudaStreamQuery(h->stream);
      if (q != cudaErrorNotReady) kernel_done = true;            // finished (or failed: reported by the synchronize below)
      else std::this_thread::yield();
    }
  }
  if (out->PF) {
    long long n = (long long)T * rr;
    L(k_unpack_psf, (int)std::min<long long>((n + 255) / 256, 1024), batch, 256, 0, d.PsF, T, r, d.PF);
    cudaMemcpyAsync(out->PF, d.PF, B * T * rr * sizeof(double), cudaMemcpyDeviceToHost, h->stream);
  }
  std::vector<int> hstat(B);
  CK(cudaMemcpyAsync(hstat.data(), d.stat, B * sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  cudaEventRecord(ev_k, h->stream);
  cudaStreamSynchronize(h->d2h_stream);
  cudaError_t e1 = cudaStreamSynchronize(cs), e2 = cudaStreamSynchronize(h->stream);
  cudaEventDestroy(ev0); cudaEventDestroy(ev_k);
  if (e1 != cudaSuccess || e2 != cudaSuccess) CK(e1 != cudaSuccess ? e1 : e2);
  bool failed = false;
  for (size_t bb = 0; bb < B; ++bb) failed = failed || hstat[bb] == 3;
  if (failed) {                                                // NaN log-likelihood somewhere: missing data or a numerical failure?
    CK(cudaMemsetAsync(d.flag, 0, sizeof(int), h->stream));
    L(k_em_scan_fused, N, batch, 64, 0, d.X, d.L, d.R, T, N, r, d.flag);      // (X only matters: Lam/R of failed panels are NaN anyway)
    int hflag = 0;
    CK(cudaMemcpyAsync(&hflag, d.flag, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    *fallback = hflag != 0;
  }
  if (!*fallback) CK(cudaGetLastError());
  return DFM_OK;
}
#endif

extern "C" {

int dfm_version(void) { return DFM_VERSION; }

const char* dfm_status_string(int s) {
  switch (s) {
    case DFM_OK: return "ok";
    case DFM_ERR_ARG: return "bad argument";
    case DFM_ERR_TOO_FEW_OBS: return "too few observations";
    case DFM_ERR_NOT_PD: return "matrix not positive definite";
    case DFM_ERR_NOT_CONVERGED: return "not converged (max_iter reached)";
    case DFM_ERR_CUDA: return "CUDA error / no device";
    case DFM_ERR_UNSUPPORTED: return "unsupported problem size";
    case DFM_ERR_NCCL: return "NCCL error";
  }
  return "unknown";
}

// release everything a handle owns (also the error paths of dfm_create_on_stream: nothing leaks)
static void handle_teardown(dfm_handle* h) {
  if (!h) return;
  if (h->stream) cudaStreamSynchronize(h->stream);
  if (h->ws) cudaFree(h->ws);
  if (h->own_stream && h->stream) cudaStreamDestroy(h->stream);
#ifndef DFM_EMU
  if (h->copy_stream) { cudaStreamSynchronize(h->copy_stream); cudaStreamDestroy(h->copy_stream); }
  if (h->pinned_one) cudaFreeHost(h->pinned_one);
  if (h->d2h_stream) { cudaStreamSynchronize(h->d2h_stream); cudaStreamDestroy(h->d2h_stream); }
  if (h->done_host) cudaFreeHost(h->done_host);
  if (h->prof) for (auto& r : *h->prof) { cudaEventDestroy(r.e0); cudaEventDestroy(r.e1); }       // events of profiled launches
#endif
  delete h->prof;
  delete h;
}

int dfm_create_on_stream(int device, void* cuda_stream, dfm_handle** out) {
  if (!out) return DFM_ERR_ARG;
  *out = nullptr;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0 || device < 0 || device >= ndev) return DFM_ERR_CUDA;
  if (cudaSetDevice(device) != cudaSuccess) return DFM_ERR_CUDA;
  dfm_handle* h = new (std::nothrow) dfm_handle();
  if (!h) return DFM_ERR_CUDA;
  h->device = device; h->ws = nullptr; h->ws_bytes = 0; h->launches = 0; h->err[0] = 0;
  h->nsm = 132;                // H100 SXM; the CUDA build reads the device's values below (the emulation build has no device)
  h->l2_bytes = 50 << 20;
  h->profile = 0; h->prof = new std::vector<ProfRec>();
  h->stream = nullptr; h->own_stream = false;
  h->copy_stream = nullptr; h->pinned_one = nullptr; h->d2h_stream = nullptr; h->done_host = nullptr; h->done_dev = nullptr; h->done_cap = 0;
#ifndef DFM_EMU
  if (cudaDeviceGetAttribute(&h->nsm, cudaDevAttrMultiProcessorCount, device) != cudaSuccess || h->nsm <= 0) { handle_teardown(h); return DFM_ERR_CUDA; }
  if (cudaDeviceGetAttribute(&h->l2_bytes, cudaDevAttrL2CacheSize, device) != cudaSuccess) { handle_teardown(h); return DFM_ERR_CUDA; }
  if (cudaStreamCreateWithFlags(&h->copy_stream, cudaStreamNonBlocking) != cudaSuccess) { h->copy_stream = nullptr; handle_teardown(h); return DFM_ERR_CUDA; }
  if (cudaStreamCreateWithFlags(&h->d2h_stream, cudaStreamNonBlocking) != cudaSuccess) { h->d2h_stream = nullptr; handle_teardown(h); return DFM_ERR_CUDA; }
  if (cudaHostAlloc((void**)&h->pinned_one, sizeof(int), cudaHostAllocDefault) != cudaSuccess) { h->pinned_one = nullptr; handle_teardown(h); return DFM_ERR_CUDA; }
  *h->pinned_one = 1;
#endif
  if (cuda_stream) { h->stream = (cudaStream_t)cuda_stream; h->own_stream = false; }
  else { if (cudaStreamCreate(&h->stream) != cudaSuccess) { h->stream = nullptr; handle_teardown(h); return DFM_ERR_CUDA; } h->own_stream = true; }
  DFM_SET_SMEM(k_em_filter_smooth, kMaxSmem); DFM_SET_SMEM(k_als_factor, kMaxSmem); DFM_SET_SMEM(k_em_contract, kMaxSmem);
  DFM_SET_SMEM(k_lyapunov, kMaxSmem); DFM_SET_SMEM(k_var, kMaxSmem); DFM_SET_SMEM(k_pca_finish, kMaxSmem);
  DFM_SET_SMEM(k_jacobi, kMaxSmem); DFM_SET_SMEM(k_subspace_eig, kMaxSmem); DFM_SET_SMEM(k_loading, kMaxSmem); DFM_SET_SMEM(k_als_lambda, kMaxSmem);
  if (cudaGetLastError() != cudaSuccess) { handle_teardown(h); return DFM_ERR_CUDA; }
  *out = h;
  return DFM_OK;
}
int dfm_create(int device, dfm_handle** out) { return dfm_create_on_stream(device, nullptr, out); }

int dfm_destroy(dfm_handle* h) {
  if (!h) return DFM_ERR_ARG;
  cudaSetDevice(h->device);
  handle_teardown(h);
  return DFM_OK;
}
int dfm_sync(dfm_handle* h) { if (!h) return DFM_ERR_ARG; CK(cudaStreamSynchronize(h->stream)); return DFM_OK; }
long long dfm_launch_count(const dfm_handle* h) { return h ? h->launches : -1; }
const char* dfm_last_error(const dfm_handle* h) { return h ? h->err : "null handle"; }

// ---- per-kernel CUDA-event profiling (bench.py's roofline leg; off by default) -----------------
int dfm_profile_enable(dfm_handle* h, int on) {
  if (!h) return DFM_ERR_ARG;
  h->profile = on ? 1 : 0;
  return DFM_OK;
}
// Sum of device time (ms) and number of launches of kernel `name` since the last reset; name = NULL
// or "" sums over all kernels.  Synchronizes the stream.
int dfm_profile_query(dfm_handle* h, const char* name, double* ms, long long* count) {
  if (!h || !ms || !count) return DFM_ERR_ARG;
  *ms = 0; *count = 0;
#ifndef DFM_EMU
  CK(cudaStreamSynchronize(h->stream));
  for (auto& r : *h->prof) {
    if (name && name[0] && strcmp(name, r.name) != 0) continue;
    float t = 0; cudaEventElapsedTime(&t, r.e0, r.e1); *ms += t; *count += 1;
  }
#endif
  return DFM_OK;
}
int dfm_profile_reset(dfm_handle* h) {
  if (!h) return DFM_ERR_ARG;
#ifndef DFM_EMU
  cudaStreamSynchronize(h->stream);
  for (auto& r : *h->prof) { cudaEventDestroy(r.e0); cudaEventDestroy(r.e1); }
#endif
  h->prof->clear();
  return DFM_OK;
}
// name of the i-th distinct profiled kernel (NULL when i is out of range)
const char* dfm_profile_kernel_name(dfm_handle* h, int i) {
  if (!h) return nullptr;
  std::vector<const char*> names;
  for (auto& r : *h->prof) { bool seen = false; for (auto n : names) if (!strcmp(n, r.name)) seen = true; if (!seen) names.push_back(r.name); }
  return (i >= 0 && i < (int)names.size()) ? names[i] : nullptr;
}

int dfm_shard_range(long long n_rep, int rank, int world, long long* begin, long long* end) {
  if (n_rep < 0 || world <= 0 || rank < 0 || rank >= world || !begin || !end) return DFM_ERR_ARG;
  *begin = n_rep * rank / world; *end = n_rep * (rank + 1) / world;
  return DFM_OK;
}

// ------------------------------------------------------------------------------------ a2
int dfm_standardize(dfm_handle* h, const double* X, int T, int N, int batch, int mem, double* Xs, double* xmean,
                    double* xstd) {
  if (!h || !X || !Xs || T <= 0 || N <= 0 || batch <= 0) return fail(h, DFM_ERR_ARG, "dfm_standardize: bad argument");
  if (batch > kMaxGridBatch) return fail(h, DFM_ERR_UNSUPPORTED, "dfm_standardize: batch > 65535");
  CK(cudaSetDevice(h->device));
  size_t B = batch, TN = (size_t)T * N;
  for (int pass = 0; pass < 2; ++pass) {
    Arena a(pass ? h->ws : nullptr);
    double* dX = mem == DFM_MEM_HOST ? a.get<double>(B * TN) : nullptr;
    double* dXs = mem == DFM_MEM_HOST ? a.get<double>(B * TN) : Xs;
    double* dm = a.get<double>(B * N); double* ds = a.get<double>(B * N);
    if (!pass) { int rc = ensure_ws(h, a.off); if (rc) return rc; continue; }
    const double* x; int rc = stage_in(h, X, dX, B * TN, mem, &x); if (rc) return rc;
    L(k_standardize, N, batch, 128, 48 * 8, x, T, N, dXs, dm, ds, (double*)nullptr, (int*)nullptr);
    if (mem == DFM_MEM_HOST) { rc = copy_out(h, Xs, dXs, B * TN, mem); if (rc) return rc; }
    rc = copy_out(h, xmean, dm, B * N, mem); if (rc) return rc;
    rc = copy_out(h, xstd, ds, B * N, mem); if (rc) return rc;
  }
  return finish(h, mem);
}

// ------------------------------------------------------------------------------------ PCA helper
// device-side PCA of the balanced columns of dXs into dF.  min(N,T) <= 64: direct Jacobi on the Gram
// matrix; larger: block subspace iteration with Rayleigh-Ritz (Ysub = scratch nmax x PCA_MMAX per panel).
#define PCA_MMAX 64
static int pca_block(int r) { return std::min(PCA_MMAX, std::max(2 * r, r + 16)); }
static int run_pca(dfm_handle* h, const double* dXs, int T, int N, int r, int batch, const int* col_n /*null = all cols*/,
                   int* bal_idx, int* nbal, double* G, double* V, double* Ysub, double* dF, int* status, AlsState* st) {
  int nmax = std::min(N, T);
  if (col_n) L(k_balanced_cols, batch, 1, 1, 0, col_n, T, N, bal_idx, nbal);
  else L(k_all_cols, batch, 1, 128, 0, N, bal_idx, nbal);
  const int nb16 = (nmax + 15) / 16, nblocks = nb16 * (nb16 + 1) / 2;
  L(k_gram_tc, (nblocks + 7) / 8, batch, 256, 0, dXs, T, N, bal_idx, nbal, G, nmax);
  if (nmax <= 64) L(k_jacobi, batch, 1, 256, (size_t)(2 * nmax * nmax + 2 * (nmax + 3) + 48) * 8, G, V, nbal, T, nmax, 60, (int*)nullptr);
  else {
    int m = std::min(nmax, pca_block(r));
    const size_t sm2 = subspace2_smem_doubles(nmax, m) * 8;
    if (sm2 <= 110 * 1024 && m <= 48) {       // iterate in shared memory, products on the tensor path
      // (one CTA per SM, to keep the resident panels' Gram matrices inside L2, was slower than two on the C5 shard)
      DFM_SET_SMEM(k_subspace_eig2, sm2);
      L(k_subspace_eig2, batch, 1, 256, sm2, G, V, nbal, T, nmax, r, m, 500, 1e-13, (int*)nullptr);
    } else L(k_subspace_eig, batch, 1, 256, (size_t)(3 * m * m + 3 * m + 72) * 8, G, V, Ysub, nbal, T, nmax, r, m, 500, 1e-13, (int*)nullptr);
  }
  {
    const size_t smF = (size_t)(r / 2 + 2 + 48 + N) * 8, smFast = (size_t)(r / 2 + 2 + 48) * 8 + (size_t)em_lds(nmax) * r * 8 + 64;
    if (N <= T && r <= 48 && smFast <= 100 * 1024)
      L(k_pca_finish, batch, 1, 256, std::max(smF, smFast), dXs, T, N, bal_idx, nbal, G, V, nmax, r, dF, status, st, 1);
    else L(k_pca_finish, batch, 1, 128, smF, dXs, T, N, bal_idx, nbal, G, V, nmax, r, dF, status, st, 0);
  }
  return DFM_OK;
}

int dfm_pca_score(dfm_handle* h, const double* X, int T, int N, int r, int batch, int mem, double* score) {
  if (!h || !X || !score || T <= 0 || N <= 0 || r <= 0 || batch <= 0 || r > std::min(T, N)) return fail(h, DFM_ERR_ARG, "dfm_pca_score: bad argument");
  if (r > 48) return fail(h, DFM_ERR_UNSUPPORTED, "dfm_pca_score: r > 48");
  if (batch > kMaxGridBatch) return fail(h, DFM_ERR_UNSUPPORTED, "dfm_pca_score: batch > 65535");
  CK(cudaSetDevice(h->device));
  size_t B = batch, TN = (size_t)T * N; int nmax = std::min(N, T);
  for (int pass = 0; pass < 2; ++pass) {
    Arena a(pass ? h->ws : nullptr);
    double* dX = mem == DFM_MEM_HOST ? a.get<double>(B * TN) : nullptr;
    double* dF = mem == DFM_MEM_HOST ? a.get<double>(B * T * r) : score;
    int* bal = a.get<int>(B * N); int* nbal = a.get<int>(B); int* status = a.get<int>(B);
    double* G = a.get<double>(B * nmax * nmax); double* V = a.get<double>(B * nmax * nmax);
    double* Ysub = a.get<double>(B * nmax * PCA_MMAX);
    if (!pass) { int rc = ensure_ws(h, a.off); if (rc) return rc; continue; }
    const double* x; int rc = stage_in(h, X, dX, B * TN, mem, &x); if (rc) return rc;
    CK(cudaMemsetAsync(status, 0, B * sizeof(int), h->stream));
    rc = run_pca(h, x, T, N, r, batch, nullptr, bal, nbal, G, V, Ysub, dF, status, nullptr); if (rc) return rc;
    if (mem == DFM_MEM_HOST) { rc = copy_out(h, score, dF, B * T * r, mem); if (rc) return rc; }
  }
  return finish(h, mem);
}

// ------------------------------------------------------------------------------------ a7
int dfm_estimate_factor(dfm_handle* h, const double* X, const dfm_factor_opts* o, const double* F_init, double* F,
                        double* Lambda, double* R2, double* xmean, double* xstd, dfm_factor_stats* stats) {
  if (!h || !X || !o) return fail(h, DFM_ERR_ARG, "dfm_estimate_factor: null argument");
  int T = o->T, N = o->N, r = o->r, batch = o->batch, mem = o->mem;
  if (T <= 1 || N <= 0 || r <= 0 || batch <= 0 || r > 64 || r > N || r > T || o->max_iter < 1 || o->n_constr < 0 ||
      (o->n_constr > 0 && (!o->constr_index || !o->constr_R || !o->constr_r)) || o->n_constr > 64)
    return fail(h, DFM_ERR_ARG, "dfm_estimate_factor: bad shape/options");
  if (!F_init && r > 48) return fail(h, DFM_ERR_UNSUPPORTED, "PCA init: r > 48 (pass F_init)");
  if (batch > kMaxGridBatch) return fail(h, DFM_ERR_UNSUPPORTED, "dfm_estimate_factor: batch > 65535");
  CK(cudaSetDevice(h->device));
  size_t B = batch, TN = (size_t)T * N; int nmax = std::min(N, T), np = r * (r + 1) / 2, nc = o->n_constr;
  int ntF = tpt_threads(np + r);
  int nblk = (T + ntF - 1) / ntF;
  // k_als_factor's per-thread packed systems: in shared memory up to r = 40 at the 32-thread floor of tpt_threads, in a
  // global scratch from the workspace past that (r <= 64)
  size_t smF = ((size_t)(np + r) * ntF + 48) * 8;
  const bool sys_global = smF > kMaxSmem;
  if (sys_global) smF = 48 * 8;
  for (int pass = 0; pass < 2; ++pass) {
    Arena a(pass ? h->ws : nullptr);
    double* dX = mem == DFM_MEM_HOST ? a.get<double>(B * TN) : nullptr;
    double* dXs = a.get<double>(B * TN);
    double* dm = a.get<double>(B * N); double* ds = a.get<double>(B * N); double* css = a.get<double>(B * N);
    int* cn = a.get<int>(B * N); AlsState* st = a.get<AlsState>(B);
    int* bal = a.get<int>(B * N); int* nbal = a.get<int>(B); int* active = a.get<int>(4);
    double* G = F_init ? nullptr : a.get<double>(B * nmax * nmax); double* V = F_init ? nullptr : a.get<double>(B * nmax * nmax);
    double* Ysub = F_init ? nullptr : a.get<double>(B * nmax * PCA_MMAX);
    double* dF = a.get<double>(B * T * r); double* dLam = a.get<double>(B * N * r); double* dR2 = a.get<double>(B * N);
    double* FtF = a.get<double>(B * r * r); double* LtL = a.get<double>(B * r * r); double* ssrp = a.get<double>(B * nblk);
    int* cidx = a.get<int>(nc + 1); double* cR = a.get<double>((size_t)nc * r + 1); double* cr = a.get<double>(nc + 1);
    double* gsys = sys_global ? a.get<double>(B * nblk * (size_t)(np + r) * ntF) : nullptr;
    if (!pass) { int rc = ensure_ws(h, a.off); if (rc) return rc; continue; }
    const double* x; int rc = stage_in(h, X, dX, B * TN, mem, &x); if (rc) return rc;
    if (nc > 0) {
      CK(cudaMemcpyAsync(cidx, o->constr_index, nc * sizeof(int), cudaMemcpyHostToDevice, h->stream));
      CK(cudaMemcpyAsync(cR, o->constr_R, (size_t)nc * r * sizeof(double), cudaMemcpyHostToDevice, h->stream));
      CK(cudaMemcpyAsync(cr, o->constr_r, nc * sizeof(double), cudaMemcpyHostToDevice, h->stream));
    }
    L(k_standardize, N, batch, 128, 48 * 8, x, T, N, dXs, dm, ds, css, cn);            // :339
    L(k_als_init_state, batch, 1, 128, 48 * 8, st, css, cn, N);                        // :342-343
    if (F_init) { const double* fi; rc = stage_in(h, F_init, dF, B * T * r, mem, &fi); if (rc) return rc;
                  if (fi != dF) CK(cudaMemcpyAsync(dF, fi, B * T * r * sizeof(double), cudaMemcpyDeviceToDevice, h->stream)); }
    else { rc = run_pca(h, dXs, T, N, r, batch, cn, bal, nbal, G, V, Ysub, dF, nullptr, st); if (rc) return rc; }   // :345-348
    size_t smL = (size_t)(2 * np + 2 * r + 8 + (size_t)r * nc + (size_t)nc * (nc + 1) / 2 + nc) * 8;
    long long it = 0;
    int h_active = batch;
    // balanced panels without constraints: all sweeps in ONE fused launch (TMA ring + DMMA passes)
    if (nc == 0 && als_fused2_shape_ok(T, N, r) && o->nt_min <= T) {
      std::vector<AlsState> hs(B);
      CK(cudaMemcpyAsync(hs.data(), st, B * sizeof(AlsState), cudaMemcpyDeviceToHost, h->stream));
      CK(cudaStreamSynchronize(h->stream));
      bool balanced = true;
      for (size_t b = 0; b < B; ++b) if (hs[b].nobs != (long long)T * N || hs[b].status != 0) balanced = false;
      if (balanced) {
        AlsFusedArgs fa{}; fa.Xs = dXs; fa.F = dF; fa.Lam = dLam; fa.st = st; fa.B = batch; fa.T = T; fa.N = N; fa.tol = o->tol; fa.max_iter = o->max_iter;
        rc = launch_als_fused2(h, fa, r); if (rc) return rc;
        h_active = 0;
      }
    }
    // panels with missing data, no constraints: all sweeps in ONE launch as well (thread-per-series / thread-per-period
    // masked normal equations, no host synchronisation in the sweep loop)
    if (h_active > 0 && nc == 0 && als_masked_shape_ok(T, N, r)) {
      AlsMaskedArgs fa{}; fa.Xs = dXs; fa.F = dF; fa.Lam = dLam; fa.st = st; fa.B = batch; fa.T = T; fa.N = N; fa.nt_min = o->nt_min;
      fa.tol = o->tol; fa.max_iter = o->max_iter;
      launch_als_masked(h, fa, r);
      h_active = 0;
    }
    while (it < o->max_iter && h_active > 0) {                                       // :352
      if (nc > 0) L(k_gram_small, batch, 1, 128, 0, dF, T, r, FtF, st);
      L(k_als_lambda, N, batch, 64, smL, dXs, dF, T, N, r, o->nt_min, 0, dLam, (double*)nullptr, FtF, nc, cidx, cR, cr, ds, st);   // :355-362
      L(k_gram_small, batch, 1, 128, 0, dLam, N, r, LtL, st);
      L(k_als_factor, nblk, batch, ntF, smF, dXs, dLam, LtL, T, N, r, dF, ssrp, st, gsys);                                           // :364-366
      L(k_als_check, batch, 1, 1, 0, st, ssrp, nblk, o->tol, T, N, o->max_iter);                                                // :367-368
      ++it;
      if ((it & 1) == 0 || it >= o->max_iter || it < 2) {
        L(k_count_active, 1, 1, 128, 48 * 8, st, batch, active);
        CK(cudaMemcpyAsync(&h_active, active, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
        CK(cudaStreamSynchronize(h->stream));
      }
    }
    if (o->compute_r2 && R2)                                                          // :372-380
      L(k_als_lambda, N, batch, 64, smL, dXs, dF, T, N, r, o->nt_min, 1, (double*)nullptr, dR2, FtF, 0, cidx, cR, cr, ds, (AlsState*)nullptr);
    rc = copy_out(h, F, dF, B * T * r, mem); if (rc) return rc;
    rc = copy_out(h, Lambda, dLam, B * N * r, mem); if (rc) return rc;
    if (o->compute_r2) { rc = copy_out(h, R2, dR2, B * N, mem); if (rc) return rc; }
    rc = copy_out(h, xmean, dm, B * N, mem); if (rc) return rc;
    rc = copy_out(h, xstd, ds, B * N, mem); if (rc) return rc;
    if (stats) {
      std::vector<AlsState> hs(B);
      CK(cudaMemcpyAsync(hs.data(), st, B * sizeof(AlsState), cudaMemcpyDeviceToHost, h->stream));
      CK(cudaStreamSynchronize(h->stream));
      for (size_t b = 0; b < B; ++b) { stats[b].ssr = hs[b].ssr; stats[b].tss = hs[b].tss; stats[b].nobs = hs[b].nobs; stats[b].iters = hs[b].iters; stats[b].status = hs[b].status; }
    }
  }
  return finish(h, mem);
}

// ------------------------------------------------------------------------------------ a9
int dfm_estimate_loading(dfm_handle* h, const double* data, const double* F, const dfm_loading_opts* o, double* lambda,
                         double* r2, double* uar_coef, double* uar_ser) {
  return dfm_estimate_loading_ex(h, data, F, o, lambda, r2, uar_coef, uar_ser, nullptr, nullptr, nullptr);
}

int dfm_estimate_loading_ex(dfm_handle* h, const double* data, const double* F, const dfm_loading_opts* o, double* lambda,
                            double* r2, double* uar_coef, double* uar_ser, double* constant, double* resid, int* status_out) {
  if (!h || !data || !F || !o) return fail(h, DFM_ERR_ARG, "dfm_estimate_loading: null argument");
  int T = o->T, ns = o->ns, r = o->r, batch = o->batch, mem = o->mem, L_ = o->n_uarlag, nc = o->n_constr;
  if (T <= 1 || ns <= 0 || r <= 0 || r > 64 || batch <= 0 || L_ <= 0 || L_ > 16 || nc < 0 || nc > 64 ||
      (nc > 0 && (!o->constr_index || !o->constr_R || !o->constr_r)))
    return fail(h, DFM_ERR_ARG, "dfm_estimate_loading: bad shape/options");
  if (batch > kMaxGridBatch) return fail(h, DFM_ERR_UNSUPPORTED, "dfm_estimate_loading: batch > 65535");
  CK(cudaSetDevice(h->device));
  size_t B = batch; int K = r + 1, np = K * (K + 1) / 2;
  for (int pass = 0; pass < 2; ++pass) {
    Arena a(pass ? h->ws : nullptr);
    double* dD = mem == DFM_MEM_HOST ? a.get<double>(B * T * ns) : nullptr;
    double* dFb = mem == DFM_MEM_HOST ? a.get<double>(B * T * r) : nullptr;
    double* dl = a.get<double>(B * ns * r); double* dr2 = a.get<double>(B * ns);
    double* dac = a.get<double>(B * ns * L_); double* dser = a.get<double>(B * ns);
    double* scr = a.get<double>(B * ns * T); int* status = a.get<int>(B);
    double* dcon = constant ? a.get<double>(B * ns) : nullptr;
    double* dres = resid ? (mem == DFM_MEM_HOST ? a.get<double>(B * ns * T) : resid) : nullptr;
    int* cidx = a.get<int>(nc + 1); double* cR = a.get<double>((size_t)nc * r + 1); double* cr = a.get<double>(nc + 1);
    if (!pass) { int rc = ensure_ws(h, a.off); if (rc) return rc; continue; }
    const double* d; const double* f;
    int rc = stage_in(h, data, dD, B * T * ns, mem, &d); if (rc) return rc;
    rc = stage_in(h, F, dFb, B * T * r, mem, &f); if (rc) return rc;
    if (nc > 0) {
      CK(cudaMemcpyAsync(cidx, o->constr_index, nc * sizeof(int), cudaMemcpyHostToDevice, h->stream));
      CK(cudaMemcpyAsync(cR, o->constr_R, (size_t)nc * r * sizeof(double), cudaMemcpyHostToDevice, h->stream));
      CK(cudaMemcpyAsync(cr, o->constr_r, nc * sizeof(double), cudaMemcpyHostToDevice, h->stream));
    }
    CK(cudaMemsetAsync(status, 0, B * sizeof(int), h->stream));
    size_t wk = std::max<size_t>((size_t)K * nc + (size_t)nc * (nc + 1) / 2 + nc, (size_t)L_ * (L_ + 1) / 2 + L_);
    size_t sm = (size_t)(np + K + 8 + wk) * 8;
    L(k_loading, ns, batch, 64, sm, d, f, T, ns, r, o->nt_min, L_, dl, dr2, dac, dser, scr, nc, cidx, cR, cr, status, dcon, dres);
    rc = copy_out(h, lambda, dl, B * ns * r, mem); if (rc) return rc;
    rc = copy_out(h, r2, dr2, B * ns, mem); if (rc) return rc;
    rc = copy_out(h, uar_coef, dac, B * ns * L_, mem); if (rc) return rc;
    rc = copy_out(h, uar_ser, dser, B * ns, mem); if (rc) return rc;
    if (constant) { rc = copy_out(h, constant, dcon, B * ns, mem); if (rc) return rc; }
    if (resid && mem == DFM_MEM_HOST) { rc = copy_out(h, resid, dres, B * ns * T, mem); if (rc) return rc; }
    if (status_out) {
      // per-panel status (0, or DFM_ERR_NOT_PD when a regression / constraint / AR step of some series was singular;
      // the affected series carry NaN).  Always a HOST array.
      CK(cudaMemcpyAsync(status_out, status, B * sizeof(int), cudaMemcpyDeviceToHost, h->stream));
      CK(cudaStreamSynchronize(h->stream));
    }
  }
  return finish(h, mem);
}

// ------------------------------------------------------------------------------------ a10
int dfm_estimate_var(dfm_handle* h, const double* F, int T, int r, int p, int withconst, int batch, int mem,
                     double* betahat, double* resid, double* seps, double* M, double* Q, double* G) {
  if (!h || !F || T <= 0 || r <= 0 || p <= 0 || batch <= 0) return fail(h, DFM_ERR_ARG, "dfm_estimate_var: bad argument");
  int k = r * p, K = k + (withconst ? 1 : 0);
  if (T - p <= K) return fail(h, DFM_ERR_TOO_FEW_OBS, "dfm_estimate_var: T - p <= K");
  size_t sm = ((size_t)K * K + (size_t)K * r + (size_t)r * r + 16) * 8 + (size_t)T + 16;
  if (sm > kMaxSmem) return fail(h, DFM_ERR_UNSUPPORTED, "dfm_estimate_var: r*p or T too large");
  CK(cudaSetDevice(h->device));
  size_t B = batch;
  for (int pass = 0; pass < 2; ++pass) {
    Arena a(pass ? h->ws : nullptr);
    double* dFb = mem == DFM_MEM_HOST ? a.get<double>(B * T * r) : nullptr;
    double* db = a.get<double>(B * K * r); double* dres = a.get<double>(B * T * r); double* dse = a.get<double>(B * r * r);
    double* dM = a.get<double>(B * k * k); double* dQ = a.get<double>(B * r * k); double* dG = a.get<double>(B * k * r);
    int* status = a.get<int>(B);
    if (!pass) { int rc = ensure_ws(h, a.off); if (rc) return rc; continue; }
    const double* f; int rc = stage_in(h, F, dFb, B * T * r, mem, &f); if (rc) return rc;
    CK(cudaMemsetAsync(status, 0, B * sizeof(int), h->stream));
    L(k_var, batch, 1, 128, sm, f, T, r, p, withconst, 0, db, dres, dse, dM, dQ, dG, (double*)nullptr, status);
    rc = copy_out(h, betahat, db, B * K * r, mem); if (rc) return rc;
    rc = copy_out(h, resid, dres, B * T * r, mem); if (rc) return rc;
    rc = copy_out(h, seps, dse, B * r * r, mem); if (rc) return rc;
    rc = copy_out(h, M, dM, B * k * k, mem); if (rc) return rc;
    rc = copy_out(h, Q, dQ, B * r * k, mem); if (rc) return rc;
    rc = copy_out(h, G, dG, B * k * r, mem); if (rc) return rc;
    std::vector<int> hs(B);
    CK(cudaMemcpyAsync(hs.data(), status, B * sizeof(int), cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    // a failed panel (too few complete rows / singular regression) has NaN in all of its outputs.  A single-panel call
    // reports the failure as the return code; a batched call fails only when NO panel could be fitted, so that one
    // degenerate bootstrap draw does not void the other replications (callers test the outputs for NaN).
    size_t nfail = 0; int first = 0;
    for (size_t b = 0; b < B; ++b) if (hs[b]) { if (!nfail) first = hs[b]; ++nfail; }
    if (nfail == B) return fail(h, first, "dfm_estimate_var: regression failed");
  }
  return finish(h, mem);
}

// ------------------------------------------------------------------------------------ a11
int dfm_irf(dfm_handle* h, const double* M, const double* Q, const double* G, int k, int r, int H, int n_shock,
            const int* shock_ids, int batch, int mem, double* irf) {
  if (!h || !M || !Q || !G || !shock_ids || !irf || k <= 0 || r <= 0 || H <= 0 || n_shock <= 0 || batch <= 0)
    return fail(h, DFM_ERR_ARG, "dfm_irf: bad argument");
  for (int j = 0; j < n_shock; ++j) if (shock_ids[j] < 0 || shock_ids[j] >= r) return fail(h, DFM_ERR_ARG, "dfm_irf: shock id out of range");
  if (batch > kMaxGridBatch) return fail(h, DFM_ERR_UNSUPPORTED, "dfm_irf: batch > 65535");
  CK(cudaSetDevice(h->device));
  size_t B = batch;
  for (int pass = 0; pass < 2; ++pass) {
    Arena a(pass ? h->ws : nullptr);
    double* dM = mem == DFM_MEM_HOST ? a.get<double>(B * k * k) : nullptr;
    double* dQ = mem == DFM_MEM_HOST ? a.get<double>(B * r * k) : nullptr;
    double* dG = mem == DFM_MEM_HOST ? a.get<double>(B * k * r) : nullptr;
    double* dI = mem == DFM_MEM_HOST ? a.get<double>(B * r * H * n_shock) : irf;
    int* ids = a.get<int>(n_shock);
    if (!pass) { int rc = ensure_ws(h, a.off); if (rc) return rc; continue; }
    const double *m, *q, *g;
    int rc = stage_in(h, M, dM, B * k * k, mem, &m); if (rc) return rc;
    rc = stage_in(h, Q, dQ, B * r * k, mem, &q); if (rc) return rc;
    rc = stage_in(h, G, dG, B * k * r, mem, &g); if (rc) return rc;
    CK(cudaMemcpyAsync(ids, shock_ids, n_shock * sizeof(int), cudaMemcpyHostToDevice, h->stream));
    L(k_irf, n_shock, batch, 64, (size_t)(2 * k + 8) * 8, m, q, g, k, r, H, n_shock, ids, dI);
    if (mem == DFM_MEM_HOST) { rc = copy_out(h, irf, dI, B * r * H * n_shock, mem); if (rc) return rc; }
  }
  return finish(h, mem);
}

// ------------------------------------------------------------------------------------ a' init
int dfm_em_init_from_factors(dfm_handle* h, const double* Xs, const double* F, int T, int N, int r, int p, int batch,
                             int mem, double* Lam, double* R, double* A, double* Q) {
  if (!h || !Xs || !F || T <= 0 || N <= 0 || r <= 0 || r > 64 || p <= 0 || batch <= 0) return fail(h, DFM_ERR_ARG, "dfm_em_init_from_factors: bad argument");
  int k = r * p;
  if (T - p <= k) return fail(h, DFM_ERR_TOO_FEW_OBS, "dfm_em_init_from_factors: T - p <= r*p");
  size_t smV = ((size_t)k * k + (size_t)k * r + (size_t)r * r + 16) * 8 + (size_t)T + 16;
  if (smV > kMaxSmem) return fail(h, DFM_ERR_UNSUPPORTED, "r*p too large");
  if (batch > kMaxGridBatch) return fail(h, DFM_ERR_UNSUPPORTED, "dfm_em_init_from_factors: batch > 65535");
  CK(cudaSetDevice(h->device));
  size_t B = batch, TN = (size_t)T * N; int np = r * (r + 1) / 2;
  EmbPlan embi = emb_plan(T, N, r, batch, h->nsm);
  for (int pass = 0; pass < 2; ++pass) {
    Arena a(pass ? h->ws : nullptr);
    double* dX = mem == DFM_MEM_HOST ? a.get<double>(B * TN) : nullptr;
    double* dFb = mem == DFM_MEM_HOST ? a.get<double>(B * T * r) : nullptr;
    double* dL = a.get<double>(B * N * r); double* dR = a.get<double>(B * N);
    double* dA = a.get<double>(B * r * k); double* dQ = a.get<double>(B * r * r); double* dres = a.get<double>(B * T * r);
    int* status = a.get<int>(B);
    EmState* est = nullptr; int* miss = nullptr; double *dFtF = nullptr, *dWs = nullptr, *dlogRs = nullptr;
    if (embi.on) {
      est = a.get<EmState>(B); miss = a.get<int>(B); dFtF = a.get<double>(B * r * r); dWs = a.get<double>(B * N * r); dlogRs = a.get<double>(B * N);
      embi.Spart = a.get<double>((size_t)embi.tsM * B * N * r); embi.sxxpart = a.get<double>((size_t)embi.tsM * B * N);
      embi.Cpart = a.get<double>(B * embi.ntM * r * r); embi.counters = a.get<int>(B * (size_t)(embi.ntE + embi.ntM));
    }
    if (!pass) { int rc = ensure_ws(h, a.off); if (rc) return rc; continue; }
    const double *x, *f;
    int rc = stage_in(h, Xs, dX, B * TN, mem, &x); if (rc) return rc;
    rc = stage_in(h, F, dFb, B * T * r, mem, &f); if (rc) return rc;
    CK(cudaMemsetAsync(status, 0, B * sizeof(int), h->stream));
    size_t smL = (size_t)(2 * np + 2 * r + 8) * 8;
    if (embi.on) {
      // balanced panels: Lam = (X'F)(F'F)^-1, R = ssr / T on the tensor-core M-step kernel (S_ff = F'F, no state covariance);
      // panels with missing data keep the masked per-series regressions
      CK(cudaMemsetAsync(est, 0, B * sizeof(EmState), h->stream));
      CK(cudaMemsetAsync(miss, 0, B * sizeof(int), h->stream));
      CK(cudaMemsetAsync(embi.counters, 0, sizeof(int) * B * (size_t)(embi.ntE + embi.ntM), h->stream));
      CK(cudaMemsetAsync(dL, 0, B * N * r * sizeof(double), h->stream));
      CK(cudaMemsetAsync(dR, 0, B * N * sizeof(double), h->stream));
      L(k_emb_init_flags, N, batch, 64, 0, x, T, N, est, miss);
      L(k_gram_small, batch, 1, 128, 0, f, T, r, dFtF, (const AlsState*)nullptr);
      emb_launch_M(h, embi, x, f, dFtF, T, N, r, batch, dL, dR, dWs, dlogRs, est);
      L(k_als_lambda, N, batch, 64, smL, x, f, T, N, r, 0, 2, dL, dR, (const double*)nullptr, 0, (const int*)nullptr,
        (const double*)nullptr, (const double*)nullptr, (const double*)nullptr, (AlsState*)nullptr, (const int*)miss);
    } else
    L(k_als_lambda, N, batch, 64, smL, x, f, T, N, r, 0, 2, dL, dR, (const double*)nullptr, 0, (const int*)nullptr,
      (const double*)nullptr, (const double*)nullptr, (const double*)nullptr, (AlsState*)nullptr, (const int*)nullptr);
    L(k_var, batch, 1, 128, smV, f, T, r, p, 0, 1, (double*)nullptr, dres, dQ, (double*)nullptr, (double*)nullptr,
      (double*)nullptr, dA, status);
    rc = copy_out(h, Lam, dL, B * N * r, mem); if (rc) return rc;
    rc = copy_out(h, R, dR, B * N, mem); if (rc) return rc;
    rc = copy_out(h, A, dA, B * r * k, mem); if (rc) return rc;
    rc = copy_out(h, Q, dQ, B * r * r, mem); if (rc) return rc;
  }
  return finish(h, mem);
}

// ------------------------------------------------------------------------------------ a'
int dfm_em_kalman(dfm_handle* h, const double* X, const dfm_em_opts* o, const dfm_em_init* init, const dfm_em_out* out) {
  if (!h || !X || !o || !init || !out || !init->Lam || !init->R || !init->A || !init->Q)
    return fail(h, DFM_ERR_ARG, "dfm_em_kalman: null argument");
  int T = o->T, N = o->N, r = o->r, p = o->p, batch = o->batch, mem = o->mem, mi = o->max_iter;
  if (T <= 1 || N <= 0 || r <= 0 || r > 64 || p <= 0 || batch <= 0 || mi <= 0 || o->tol < 0)
    return fail(h, DFM_ERR_ARG, "dfm_em_kalman: bad shape/options");
  if (batch > kMaxGridBatch) return fail(h, DFM_ERR_UNSUPPORTED, "dfm_em_kalman: batch > 65535");
  const int stgT = fs_stage_periods(h->nsm, batch, r, p);
  size_t smFS = em_fs_smem_doubles(r, p, stgT) * 8;
  if (smFS > kMaxSmem) return fail(h, DFM_ERR_UNSUPPORTED, "dfm_em_kalman: state dimension r*p too large for the general path");
  CK(cudaSetDevice(h->device));
  size_t B = batch, TN = (size_t)T * N; int k = r * p, kk = k * k, rr = r * r, rk = r * k, np = r * (r + 1) / 2;
  const bool fused_ok = fused_shape_ok(T, N, r, p);
  if (o->path == 2 && !fused_ok) return fail(h, DFM_ERR_UNSUPPORTED, "dfm_em_kalman: fused path needs p = 1, r <= 8 and a panel that fits shared memory");
  const bool fused2_ok = fused2_shape_ok(T, N, r, p);
  if (o->path == 3 && !fused2_ok) return fail(h, DFM_ERR_UNSUPPORTED, "dfm_em_kalman: TMA fused path needs p = 1, r <= 8, even T and a panel that fits shared memory");
  const bool try_fused = (fused_ok || fused2_ok) && o->path != 1;      // the path is only chosen after the NaN scan
  const bool use2 = fused2_ok && (o->path == 0 || o->path == 3);
  const EmbPlan emb = emb_plan(T, N, r, batch, h->nsm);
  for (int pass = 0; pass < 2; ++pass) {
    Arena a(pass ? h->ws : nullptr);
    EmBufs d;
    d.X = mem == DFM_MEM_HOST ? a.get<double>(B * TN) : nullptr;
    d.L = a.get<double>(B * N * r); d.R = a.get<double>(B * N);
    d.A = a.get<double>(B * rk); d.Q = a.get<double>(B * rr); d.P0 = a.get<double>(B * kk);
    d.Fs = a.get<double>(B * T * r); d.PsF = a.get<double>(B * T * np);
    d.ll = a.get<double>(B * mi); d.st = a.get<EmState>(B);
    d.it = a.get<int>(B); d.stat = a.get<int>(B); d.active = a.get<int>(4);
    d.PF = out->PF ? a.get<double>(B * T * rr) : nullptr;
    d.flag = a.get<int>(4);
    d.ready = a.get<int>(kMaxReadyChunks);
    d.scratch = try_fused ? a.get<double>((size_t)std::min(batch, h->nsm * 8) * T * FUSED_SCR(r)) : nullptr;
    const GenBufs g = gen_bufs(a, emb, B, T, N, r, p);        // also the fallback when the scan finds missing data
    if (!pass) { int rc = ensure_ws(h, a.off); if (rc) return rc; continue; }
    int rc = DFM_OK;
    bool fused = try_fused;
    bool uploaded = false;                // the streaming host path found missing data: the panels are on the device already
#ifndef DFM_EMU
    if (mem == DFM_MEM_HOST && use2 && em_streaming_applies(h, o)) {
      rc = em_streaming(h, X, o, init, out, d, &uploaded);
      if (rc || !uploaded) return rc;
      if (o->path == 3) return fail(h, DFM_ERR_UNSUPPORTED, "dfm_em_kalman: fused path needs a balanced panel (no NaN)");
      fused = false;                      // general path on the whole batch (the fused kernel updated earlier chunks in place)
    }
#endif
    const double* x = d.X;
    if (!uploaded) { rc = stage_in(h, X, d.X, B * TN, mem, &x); if (rc) return rc; }
    cudaMemcpyKind kin = mem == DFM_MEM_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
    CK(cudaMemcpyAsync(d.L, init->Lam, B * N * r * 8, kin, h->stream));
    CK(cudaMemcpyAsync(d.R, init->R, B * N * 8, kin, h->stream));
    CK(cudaMemcpyAsync(d.A, init->A, B * rk * 8, kin, h->stream));
    CK(cudaMemcpyAsync(d.Q, init->Q, B * rr * 8, kin, h->stream));
    if (init->P0) CK(cudaMemcpyAsync(d.P0, init->P0, B * kk * 8, kin, h->stream));
    else L(k_lyapunov, batch, 1, 128, (size_t)(3 * kk + 8) * 8, d.A, d.Q, r, p, d.P0, 12);
    {
      long long n = (long long)B * mi;
      L(k_fill, (int)std::min<long long>((n + 255) / 256, 1024), 1, 256, 0, d.ll, n, DFM_NAN);
    }
    if (fused) {                          // balanced panel, all series in the model?
      CK(cudaMemsetAsync(d.flag, 0, sizeof(int), h->stream));
      L(k_em_scan_fused, N, batch, 64, 0, x, d.L, d.R, T, N, r, d.flag);
      int hflag = 0;
      CK(cudaMemcpyAsync(&hflag, d.flag, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
      CK(cudaStreamSynchronize(h->stream));
      if (hflag) {
        if (o->path == 2 || o->path == 3) return fail(h, DFM_ERR_UNSUPPORTED, "dfm_em_kalman: fused path needs a balanced panel (no NaN)");
        fused = false;
      }
    }
    if (fused) rc = launch_em_fused(h, fused_args(d, o, x), r, use2);
    else rc = run_em_general(h, x, o, d, g, out->PF ? 1 : 0);
    if (rc) return rc;
    rc = copy_out(h, out->Lam, d.L, B * N * r, mem); if (rc) return rc;
    rc = copy_out(h, out->R, d.R, B * N, mem); if (rc) return rc;
    rc = copy_out(h, out->A, d.A, B * rk, mem); if (rc) return rc;
    rc = copy_out(h, out->Q, d.Q, B * rr, mem); if (rc) return rc;
    rc = copy_out(h, out->P0, d.P0, B * kk, mem); if (rc) return rc;
    rc = copy_out(h, out->F, d.Fs, B * T * r, mem); if (rc) return rc;
    if (out->PF) {
      long long n = (long long)T * rr;
      L(k_unpack_psf, (int)std::min<long long>((n + 255) / 256, 1024), batch, 256, 0, d.PsF, T, r, d.PF);
      rc = copy_out(h, out->PF, d.PF, B * T * rr, mem); if (rc) return rc;
    }
    rc = copy_out(h, out->loglik, d.ll, B * mi, mem); if (rc) return rc;
    rc = copy_out(h, out->iters, d.it, B, mem); if (rc) return rc;
    rc = copy_out(h, out->status, d.stat, B, mem); if (rc) return rc;
  }
  return finish(h, mem);
}

// ------------------------------------------------------------------------------------ a'': smoothing / nowcasting / forecasting
// One E-step of the general path at fixed parameters on panels padded with H all-missing periods (ss_estep), shared by
// dfm_kalman_smooth (then k_ss_project) and dfm_simulation_smoother (then the k_sim_* kernels).  Nothing here writes the
// parameter buffers: k_em_prep runs only in its opening mode (W, log R, C), k_em_filter_smooth's transition M-step goes to
// scratch, and no measurement M-step or closing step is launched.

// Shapes and options both entry points accept (`what`: the entry point, for the error message).
static int ss_check(dfm_handle* h, const char* what, int T, int N, int r, int p, int H, int batch, int mem) {
  char msg[128];
  if (T <= 0 || N <= 0 || r <= 0 || r > 64 || p <= 0 || H < 0 || batch <= 0 || (mem != DFM_MEM_HOST && mem != DFM_MEM_DEVICE) ||
      (long long)T + H < 2) {
    snprintf(msg, sizeof(msg), "%s: bad shape/options", what);
    return fail(h, DFM_ERR_ARG, msg);
  }
  if (batch > kMaxGridBatch) { snprintf(msg, sizeof(msg), "%s: batch > 65535", what); return fail(h, DFM_ERR_UNSUPPORTED, msg); }
  const int stgT = fs_stage_periods(h->nsm, batch, r, p);
  if (r * p > 48 || em_fs_smem_doubles(r, p, stgT) * 8 > kMaxSmem) {
    snprintf(msg, sizeof(msg), "%s: state dimension r*p too large for the general path", what);
    return fail(h, DFM_ERR_UNSUPPORTED, msg);
  }
  return DFM_OK;
}

// Device buffers of the fixed-parameter E-step over B panels of Tp = T + H periods, and the device views of its inputs.
struct SsStage {
  double *Xp, *L, *R, *A, *Q, *P0, *Fs, *PsF, *ll;
  EmState* st;
  int *it, *stat;
  GenBufs g;
  const double *x, *pL, *pR, *pA, *pQ;            // padded panels and parameters on the device (set by ss_estep)
};
static SsStage ss_bufs(Arena& a, int mem, int H, size_t B, int Tp, int N, int r, int p) {
  const size_t TN = (size_t)Tp * N; const int k = r * p, kk = k * k, rr = r * r, rk = r * k, np = r * (r + 1) / 2;
  SsStage s{};
  // padded panel: needed unless the input is already on the device with nothing to pad
  s.Xp = (mem == DFM_MEM_HOST || H > 0) ? a.get<double>(B * TN) : nullptr;
  s.L = mem == DFM_MEM_HOST ? a.get<double>(B * N * r) : nullptr;
  s.R = mem == DFM_MEM_HOST ? a.get<double>(B * N) : nullptr;
  s.A = mem == DFM_MEM_HOST ? a.get<double>(B * rk) : nullptr;
  s.Q = mem == DFM_MEM_HOST ? a.get<double>(B * rr) : nullptr;
  s.P0 = a.get<double>(B * kk);
  s.Fs = a.get<double>(B * Tp * r); s.PsF = a.get<double>(B * Tp * np);
  s.ll = a.get<double>(B); s.st = a.get<EmState>(B);
  s.it = a.get<int>(B); s.stat = a.get<int>(B);
  s.g = gen_bufs(a, EmbPlan{}, B, Tp, N, r, p);
  return s;
}

// Staging (padded panels, parameters, P0) and one E-step of the general path's kernels; k_em_prep in its opening mode only
// reads Lam, R.  Leaves the smoothed moments in s.Fs / s.PsF / s.ll, the per-panel status in s.stat, and the filter's
// covariances, b_t, C_t and src in s.g.
static int ss_estep(dfm_handle* h, SsStage& s, const double* X, const dfm_em_init* params, int T, int N, int r, int p, int H, int batch,
                    int mem) {
  const size_t B = batch, TN = (size_t)(T + H) * N; const int Tp = T + H;
  const int k = r * p, kk = k * k, rr = r * r, rk = r * k, np = r * (r + 1) / 2;
  const int ntC = tpt_threads(np + r), nblkC = (Tp + ntC - 1) / ntC;
  int rc = DFM_OK;
  s.x = X;
  if (mem == DFM_MEM_HOST) {
    if (H > 0) {
      CK(cudaMemcpy2DAsync(s.Xp, (size_t)Tp * 8, X, (size_t)T * 8, (size_t)T * 8, B * N, cudaMemcpyHostToDevice, h->stream));
      long long n = (long long)B * N * H;
      L(k_ss_pad, (int)std::min<long long>((n + 255) / 256, 4096), 1, 256, 0, (const double*)nullptr, T, Tp, (long long)B * N, s.Xp);
    } else CK(cudaMemcpyAsync(s.Xp, X, B * TN * 8, cudaMemcpyHostToDevice, h->stream));
    s.x = s.Xp;
  } else if (H > 0) {
    long long n = (long long)B * TN;
    L(k_ss_pad, (int)std::min<long long>((n + 255) / 256, 4096), 1, 256, 0, X, T, Tp, (long long)B * N, s.Xp);
    s.x = s.Xp;
  }
  rc = stage_in(h, params->Lam, s.L, B * N * r, mem, &s.pL); if (rc) return rc;
  rc = stage_in(h, params->R, s.R, B * N, mem, &s.pR); if (rc) return rc;
  rc = stage_in(h, params->A, s.A, B * rk, mem, &s.pA); if (rc) return rc;
  rc = stage_in(h, params->Q, s.Q, B * rr, mem, &s.pQ); if (rc) return rc;
  if (params->P0) CK(cudaMemcpyAsync(s.P0, params->P0, B * kk * 8, mem == DFM_MEM_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, h->stream));
  else L(k_lyapunov, batch, 1, 128, (size_t)(3 * kk + 8) * 8, s.pA, s.pQ, r, p, s.P0, 12);
  L(k_em_state_init, batch, 1, 1, 0, s.st);
  L(k_em_scan, N, batch, 64, 0, s.x, s.pL, Tp, N, r, s.st);
  L(k_em_prep, batch, 1, 128, 0, s.pL, s.pR, N, r, p, s.g.W, s.g.logR, s.g.C, (double*)nullptr, (const double*)nullptr, (double*)nullptr,
    (const double*)nullptr, s.st, 1, 0, 0);
  L(k_em_contract, nblkC, batch, ntC, ((size_t)(np + r) * ntC + 8) * 8, s.x, s.pL, s.g.W, s.pR, s.g.logR, s.g.C, Tp, N, r, s.g.Bt, s.g.qt,
    s.g.slr, s.g.nt, s.g.Ct, s.st);
  L(k_em_contract_bal, (Tp + 31) / 32, batch, 256, 8 * 32 * 3 * 8, s.x, s.g.W, s.pR, s.g.logR, Tp, N, r, s.g.Bt, s.g.qt, s.g.slr, s.g.nt, s.st);
  int ncl = fs_cluster_size(h, batch, s.g.xch);
  rc = launch_filter_smooth(h, ncl, s.g, batch, Tp, r, p, s.pA, s.pQ, s.P0, s.Fs, s.PsF, s.ll, s.st, 1, 0.0, 1);
  if (rc) return rc;
  L(k_em_collect, batch, 1, 1, 0, s.st, s.it, s.stat);
  return DFM_OK;
}

int dfm_kalman_smooth(dfm_handle* h, const double* X, const dfm_ss_opts* o, const dfm_em_init* params, const dfm_ss_out* out) {
  if (!h || !X || !o || !params || !out || !params->Lam || !params->R || !params->A || !params->Q)
    return fail(h, DFM_ERR_ARG, "dfm_kalman_smooth: null argument");
  const int T = o->T, N = o->N, r = o->r, p = o->p, H = o->H, batch = o->batch, mem = o->mem;
  int rc = ss_check(h, "dfm_kalman_smooth", T, N, r, p, H, batch, mem);
  if (rc) return rc;
  const int Tp = T + H;
  const size_t smP = ss_project_smem_doubles(r) * 8;
  CK(cudaSetDevice(h->device));
  const size_t B = batch, TN = (size_t)Tp * N; const int rr = r * r;
  const bool dev_out = mem == DFM_MEM_DEVICE;
  for (int pass = 0; pass < 2; ++pass) {
    Arena a(pass ? h->ws : nullptr);
    SsStage s = ss_bufs(a, mem, H, B, Tp, N, r, p);
    double* dPFfull = (out->PF && !dev_out) ? a.get<double>(B * Tp * rr) : nullptr;
    double* dcom = (out->common && !dev_out) ? a.get<double>(B * TN) : nullptr;
    double* dxh = (out->xhat && !dev_out) ? a.get<double>(B * TN) : nullptr;
    double* dxv = (out->xvar && !dev_out) ? a.get<double>(B * TN) : nullptr;
    if (!pass) { rc = ensure_ws(h, a.off); if (rc) return rc; continue; }
    rc = ss_estep(h, s, X, params, T, N, r, p, H, batch, mem);
    if (rc) return rc;
    L(k_ss_nan_failed, batch, 1, 256, 0, (const EmState*)s.st, Tp, r, s.Fs, s.PsF, s.ll);
    // ---- projection onto the series
    double* ocom = dev_out ? out->common : dcom;
    double* oxh = dev_out ? out->xhat : dxh;
    double* oxv = dev_out ? out->xvar : dxv;
    if (ocom || oxh || oxv) {
      DFM_SET_SMEM(k_ss_project, smP);
      const int nst = (N + SS_NS - 1) / SS_NS, ntt = (Tp + SS_TP - 1) / SS_TP;
      const int per = std::max(1, 65535 / nst);            // panels per launch (grid.y limit)
      for (int b0 = 0; b0 < batch; b0 += per) {
        const int nb = std::min(per, batch - b0);
        L(k_ss_project, ntt, nst * nb, 256, smP, s.x, (const double*)s.Fs, (const double*)s.PsF, s.pL, s.pR, (const EmState*)s.st, Tp, N, r,
          b0, ocom, oxh, oxv);
      }
    }
    // ---- results
    rc = copy_out(h, out->F, s.Fs, B * Tp * r, mem); if (rc) return rc;
    if (out->PF) {
      long long n = (long long)Tp * rr;
      double* dst = dev_out ? out->PF : dPFfull;
      L(k_unpack_psf, (int)std::min<long long>((n + 255) / 256, 1024), batch, 256, 0, s.PsF, Tp, r, dst);
      if (!dev_out) { rc = copy_out(h, out->PF, dPFfull, B * Tp * rr, mem); if (rc) return rc; }
    }
    if (!dev_out) {
      rc = copy_out(h, out->common, dcom, B * TN, mem); if (rc) return rc;
      rc = copy_out(h, out->xhat, dxh, B * TN, mem); if (rc) return rc;
      rc = copy_out(h, out->xvar, dxv, B * TN, mem); if (rc) return rc;
    }
    rc = copy_out(h, out->loglik, s.ll, B, mem); if (rc) return rc;
    rc = copy_out(h, out->status, s.stat, B, mem); if (rc) return rc;
  }
  return finish(h, mem);
}

// ------------------------------------------------------------------------------------ simulation smoother
// Draws per chunk: the per-draw scratch of k_sim_paths (zf_t and f+_t of every period) and, for host outputs, the staging of
// one chunk's draws stay within kSimChunkBytes whatever n_draw; k_sim_project's grid.y (<= 65535) bounds the chunk as well.
static const size_t kSimChunkBytes = (size_t)512 << 20;
static long long sim_chunk(long long n_draw, int Tp, int N, int r, int k, bool stageF, bool stageX) {
  const size_t per = (size_t)Tp * (k + r + (stageF ? r : 0) + (stageX ? N : 0)) * 8;
  long long c = (long long)std::max<size_t>(SIM_ND, kSimChunkBytes / per);
  c = std::min<long long>(c, (long long)(65535 / ((N + SS_NS - 1) / SS_NS)) * SIM_PD);
  return std::min(c, n_draw);
}

// The E-step of dfm_kalman_smooth (one model), k_sim_gains once, then k_sim_paths (and k_sim_project when panel draws are
// requested) per chunk of draws.
int dfm_simulation_smoother(dfm_handle* h, const double* X, const dfm_sim_opts* o, const dfm_em_init* params, const dfm_sim_out* out) {
  if (!h || !X || !o || !params || !out || !params->Lam || !params->R || !params->A || !params->Q)
    return fail(h, DFM_ERR_ARG, "dfm_simulation_smoother: null argument");
  const int T = o->T, N = o->N, r = o->r, p = o->p, H = o->H, mem = o->mem;
  if (o->n_draw < 1 || o->draw0 < 0) return fail(h, DFM_ERR_ARG, "dfm_simulation_smoother: n_draw < 1 or draw0 < 0");
  int rc = ss_check(h, "dfm_simulation_smoother", T, N, r, p, H, 1, mem);
  if (rc) return rc;
  const int Tp = T + H, k = r * p;
  const size_t smG = sim_gains_smem_doubles(r, p) * 8, smS = sim_paths_smem_doubles(r, p) * 8, smP = sim_project_smem_doubles(r) * 8;
  CK(cudaSetDevice(h->device));
  const bool dev_out = mem == DFM_MEM_DEVICE;
  const long long nch = sim_chunk(o->n_draw, Tp, N, r, k, out->F && !dev_out, out->X && !dev_out);
  for (int pass = 0; pass < 2; ++pass) {
    Arena a(pass ? h->ws : nullptr);
    SsStage s = ss_bufs(a, mem, H, 1, Tp, N, r, p);
    double* gains = a.get<double>(sim_gains_doubles(Tp, k, r));
    int* sstat = a.get<int>(1);
    double* zfS = a.get<double>((size_t)nch * Tp * k);
    double* fS = a.get<double>((size_t)nch * Tp * r);
    double* dF = (out->F && !dev_out) ? a.get<double>((size_t)nch * Tp * r) : nullptr;
    double* dX = (out->X && !dev_out) ? a.get<double>((size_t)nch * Tp * N) : nullptr;
    if (!pass) { rc = ensure_ws(h, a.off); if (rc) return rc; continue; }
    rc = ss_estep(h, s, X, params, T, N, r, p, H, 1, mem);
    if (rc) return rc;
    const int* src = s.g.nt + Tp;                        // src[t] of k_em_filter_smooth (g.nt: n_t, then src_t)
    CK(cudaMemsetAsync(sstat, 0, sizeof(int), h->stream));
    DFM_SET_SMEM(k_sim_gains, smG);
    L(k_sim_gains, Tp + 1, 1, 256, smG, s.pA, s.pQ, (const double*)s.P0, (const double*)s.g.C, (const double*)s.g.Ct, (const double*)s.g.Bt,
      (const double*)s.g.Pp, (const double*)s.g.Pf, src, (const int*)s.g.nt, (const EmState*)s.st, Tp, r, p, gains, sstat);
    DFM_SET_SMEM(k_sim_paths, smS);
    DFM_SET_SMEM(k_sim_project, smP);
    const int nst = (N + SS_NS - 1) / SS_NS, ntt = (Tp + SS_TP - 1) / SS_TP;
    for (long long j0 = 0; j0 < o->n_draw; j0 += nch) {
      const int nd = (int)std::min(nch, o->n_draw - j0);
      const long long id0 = o->draw0 + j0;
      double* Fo = out->F ? (dev_out ? out->F + (size_t)j0 * Tp * r : dF) : nullptr;
      double* Xo = out->X ? (dev_out ? out->X + (size_t)j0 * Tp * N : dX) : nullptr;
      L(k_sim_paths, (nd + SIM_ND - 1) / SIM_ND, 1, SIM_NT, smS, (const double*)gains, src, Tp, r, p, o->seed, id0, nd, (const int*)sstat,
        zfS, fS, Fo);
      if (Xo)
        L(k_sim_project, ntt, nst * ((nd + SIM_PD - 1) / SIM_PD), 256, smP, s.x, s.pL, s.pR, (const double*)fS, Tp, N, r, o->seed, id0, nd,
          (const int*)sstat, Xo);
      if (!dev_out) {
        if (out->F) { rc = copy_out(h, out->F + (size_t)j0 * Tp * r, dF, (size_t)nd * Tp * r, mem); if (rc) return rc; }
        if (out->X) { rc = copy_out(h, out->X + (size_t)j0 * Tp * N, dX, (size_t)nd * Tp * N, mem); if (rc) return rc; }
      }
    }
    rc = copy_out(h, out->status, sstat, 1, mem); if (rc) return rc;
  }
  return finish(h, mem);
}

// ------------------------------------------------------------------------------------ news decomposition
// The E-step of dfm_kalman_smooth on the old vintage (ss_estep), then k_news_window, k_news_cov, k_news_project and
// k_news_finish.  Only the release window of X_new is staged; for host memory the rows above it are compared with X_old
// here, so that the rest of the new panel never crosses PCIe.
int dfm_news(dfm_handle* h, const double* X_old, const double* X_new, const dfm_news_opts* o, const dfm_em_init* params,
             const dfm_news_out* out) {
  if (!h || !X_old || !X_new || !o || !params || !out || !params->Lam || !params->R || !params->A || !params->Q || !o->target_series ||
      !o->target_period)
    return fail(h, DFM_ERR_ARG, "dfm_news: null argument");
  const int T = o->T, N = o->N, r = o->r, p = o->p, H = o->H, batch = o->batch, mem = o->mem, nr = o->news_rows, nq = o->n_target;
  int rc = ss_check(h, "dfm_news", T, N, r, p, H, batch, mem);
  if (rc) return rc;
  if (nr < 1 || nr > T || nq < 1 || nq > NEWS_MAXQ) return fail(h, DFM_ERR_ARG, "dfm_news: news_rows or n_target out of range");
  const int Tp = T + H;
  std::vector<int> tg(2 * (size_t)nq), outside;        // target series, then periods; target periods outside the window
  for (int q = 0; q < nq; ++q) {
    const int i = o->target_series[q], t = o->target_period[q];
    if (i < 0 || i >= N || t < 0 || t >= Tp) return fail(h, DFM_ERR_ARG, "dfm_news: target series or period out of range");
    tg[q] = i; tg[nq + q] = t;
    if (t < T - nr || t >= T) outside.push_back(t);
  }
  std::sort(outside.begin(), outside.end());
  const int Wmax = nr + (int)(std::unique(outside.begin(), outside.end()) - outside.begin());
  if ((long long)Wmax * r > NEWS_MAXN) return fail(h, DFM_ERR_UNSUPPORTED, "dfm_news: W r > 128 (too many periods in the window and targets)");
  const bool dev = mem == DFM_MEM_DEVICE;
  const size_t B = batch, onr = (size_t)nr * N;
  std::vector<int> hbad;
  if (!dev) {                                          // the rows above the window: X_new must repeat X_old there
    hbad.assign(B, 0);
    const size_t na = (size_t)(T - nr);
    for (size_t c = 0; c < B * N && na > 0; ++c) {
      const double* x0 = X_old + c * T; const double* x1 = X_new + c * T;
      if (memcmp(x0, x1, na * sizeof(double)) == 0) continue;
      for (size_t t = 0; t < na; ++t)
        if (std::isnan(x0[t]) != std::isnan(x1[t]) || (!std::isnan(x0[t]) && x0[t] != x1[t])) { hbad[c / N] = 1; break; }
    }
  }
  const int nmax = Wmax * r;
  const size_t smW = news_window_smem_bytes(nr, nq);
  const size_t smallC = news_cov_small_doubles(r, p), bigC = news_cov_big_doubles(r, p, nmax, nq);
  const bool big_in_smem = (smallC + bigC) * 8 <= kMaxSmem;
  const size_t smC = (big_in_smem ? smallC + bigC : smallC) * 8, smP = news_project_smem_doubles(r) * 8;
  const int nst = (N + NEWS_NS - 1) / NEWS_NS, ntw = (nr + NEWS_TP - 1) / NEWS_TP, ntile = nst * ntw;
  CK(cudaSetDevice(h->device));
  for (int pass = 0; pass < 2; ++pass) {
    Arena a(pass ? h->ws : nullptr);
    SsStage s = ss_bufs(a, mem, H, B, Tp, N, r, p);
    double* dXn = dev ? nullptr : a.get<double>(B * onr);
    int* dtg = a.get<int>(2 * (size_t)nq);
    unsigned char* dmask = a.get<unsigned char>(B * onr);
    int* dpl = a.get<int>(B * (Wmax + 1));
    int* drowp = a.get<int>(B * nr);
    int* dpst = a.get<int>(B);
    int* dkind = a.get<int>(B * nq);
    double* dold = a.get<double>(B * nq);
    double* dgv = a.get<double>(B * nq * nmax);
    double* dpart = a.get<double>(B * ntile * nq);
    double* dbig = big_in_smem ? nullptr : a.get<double>(B * bigC);
    double* hOld = (out->old_est && !dev) ? a.get<double>(B * nq) : nullptr;
    double* hNew = (out->new_est && !dev) ? a.get<double>(B * nq) : nullptr;
    double* hNews = (out->news && !dev) ? a.get<double>(B * onr) : nullptr;
    double* hW = (out->weight && !dev) ? a.get<double>(B * onr * nq) : nullptr;
    double* hC = (out->contrib && !dev) ? a.get<double>(B * onr * nq) : nullptr;
    if (!pass) { rc = ensure_ws(h, a.off); if (rc) return rc; continue; }
    rc = ss_estep(h, s, X_old, params, T, N, r, p, H, batch, mem);
    if (rc) return rc;
    const int* src = s.g.nt + B * Tp;                  // src[t] of k_em_filter_smooth (g.nt: n_t, then src_t), per pair
    CK(cudaMemcpyAsync(dtg, tg.data(), tg.size() * sizeof(int), cudaMemcpyHostToDevice, h->stream));
    const double* xn = X_new; int ldn = T, row0 = T - nr;
    if (dev) CK(cudaMemsetAsync(dpst, 0, B * sizeof(int), h->stream));
    else {
      CK(cudaMemcpyAsync(dpst, hbad.data(), B * sizeof(int), cudaMemcpyHostToDevice, h->stream));
      CK(cudaMemcpy2DAsync(dXn, (size_t)nr * 8,X_new + (T - nr), (size_t)T * 8, (size_t)nr * 8, B * N, cudaMemcpyHostToDevice, h->stream));
      xn = dXn; ldn = nr; row0 = 0;
    }
    L(k_news_window, batch, 1, 256, smW, s.x, xn, ldn, row0, dev ? X_new : (const double*)nullptr, s.pL, s.pR, (const int*)dtg + nq, nq,
      (const int*)s.stat, T, Tp, N, r, nr, Wmax, dmask, dpl, drowp, dpst);
    DFM_SET_SMEM(k_news_cov, smC);
    L(k_news_cov, batch, 1, 256, smC, s.pA, (const double*)s.g.Pp, (const double*)s.g.Pf, src, (const double*)s.Fs, s.x, s.pL, s.pR,
      (const unsigned char*)dmask, (const int*)dpl, (const int*)dtg, (const int*)dtg + nq, nq, (const int*)dpst, T, Tp, N, r, p, nr, Wmax,
      dbig, dgv, dkind, dold);
    double* oNews = out->news ? (dev ? out->news : hNews) : nullptr;
    double* oW = out->weight ? (dev ? out->weight : hW) : nullptr;
    double* oC = out->contrib ? (dev ? out->contrib : hC) : nullptr;
    DFM_SET_SMEM(k_news_project, smP);
    const int per = std::max(1, 65535 / nst);          // pairs per launch (grid.y limit)
    for (int b0 = 0; b0 < batch; b0 += per) {
      const int nb = std::min(per, batch - b0);
      L(k_news_project, ntw, nst * nb, 256, smP, (const double*)s.Fs, xn, ldn, row0, s.pL, s.pR, (const unsigned char*)dmask,
        (const int*)drowp, (const double*)dgv, (const int*)dkind, (const int*)dtg, (const int*)dtg + nq, nq, (const int*)dpst, T, Tp, N, r,
        nr, Wmax, b0, oNews, oW, oC, dpart);
    }
    L(k_news_finish, batch, 1, 64, 0, (const double*)dpart, ntile, (const double*)dold, (const int*)dpst, nq,
      out->old_est ? (dev ? out->old_est : hOld) : (double*)nullptr, out->new_est ? (dev ? out->new_est : hNew) : (double*)nullptr);
    if (!dev) {
      rc = copy_out(h, out->old_est, hOld, B * nq, mem); if (rc) return rc;
      rc = copy_out(h, out->new_est, hNew, B * nq, mem); if (rc) return rc;
      rc = copy_out(h, out->news, hNews, B * onr, mem); if (rc) return rc;
      rc = copy_out(h, out->weight, hW, B * onr * nq, mem); if (rc) return rc;
      rc = copy_out(h, out->contrib, hC, B * onr * nq, mem); if (rc) return rc;
    }
    rc = copy_out(h, out->status, dpst, B, mem); if (rc) return rc;
  }
  return finish(h, mem);
}

// ------------------------------------------------------------------------------------ (e)
// ------------------------------------------------------------------------------------ K9: replication generators
int dfm_simulate_panels(dfm_handle* h, unsigned long long seed, long long rep0, int batch, int T, int N, int r, int mem,
                        double* X, double* F_true) {
  if (!h || !X || batch <= 0 || T <= 1 || N <= 0 || r <= 0 || r > 64 || rep0 < 0) return fail(h, DFM_ERR_ARG, "dfm_simulate_panels: bad argument");
  CK(cudaSetDevice(h->device));
  size_t B = batch;
  for (int pass = 0; pass < 2; ++pass) {
    Arena a(pass ? h->ws : nullptr);
    double* dX = mem == DFM_MEM_HOST ? a.get<double>(B * T * N) : X;
    double* dF = (mem == DFM_MEM_HOST || !F_true) ? a.get<double>(B * T * r) : F_true;
    if (!pass) { int rc = ensure_ws(h, a.off); if (rc) return rc; continue; }
    L(k_simulate_panels, batch, 1, 256, 0, seed, rep0, T, N, r, dX, dF);
    if (mem == DFM_MEM_HOST) { int rc = copy_out(h, X, dX, B * T * N, mem); if (rc) return rc; }
    if (F_true) { int rc = copy_out(h, F_true, dF, B * T * r, mem); if (rc) return rc; }
  }
  return finish(h, mem);
}

int dfm_bootstrap_panels(dfm_handle* h, const dfm_boot_opts* o, const double* F0, const double* resid, const double* beta,
                         const double* lam, const double* uar_coef, const double* uar_ser, const double* data, double* X) {
  if (!h || !o || !F0 || !resid || !beta || !lam || !uar_coef || !uar_ser || !data || !X)
    return fail(h, DFM_ERR_ARG, "dfm_bootstrap_panels: null argument");
  int Tw = o->T, ns = o->ns, r = o->r, p = o->p, Lg = o->n_uarlag, nres = o->n_resid, batch = o->batch, mem = o->mem;
  if (Tw <= p || ns <= 0 || r <= 0 || p <= 0 || Lg <= 0 || Lg > 16 || nres <= 0 || batch <= 0 || o->burn < 0 || o->rep0 < 0)
    return fail(h, DFM_ERR_ARG, "dfm_bootstrap_panels: bad shape/options");
  size_t smem = (size_t)Tw * r * 8;
  if (smem > kMaxSmem) return fail(h, DFM_ERR_UNSUPPORTED, "dfm_bootstrap_panels: T*r too large");
  CK(cudaSetDevice(h->device));
  size_t B = batch; int K = 1 + r * p;
  for (int pass = 0; pass < 2; ++pass) {
    Arena a(pass ? h->ws : nullptr);
    const bool hst = mem == DFM_MEM_HOST;
    double* dF0 = hst ? a.get<double>((size_t)Tw * r) : nullptr; double* dre = hst ? a.get<double>((size_t)nres * r) : nullptr;
    double* dbe = hst ? a.get<double>((size_t)K * r) : nullptr; double* dla = hst ? a.get<double>((size_t)ns * r) : nullptr;
    double* dac = hst ? a.get<double>((size_t)ns * Lg) : nullptr; double* dse = hst ? a.get<double>(ns) : nullptr;
    double* dda = hst ? a.get<double>((size_t)Tw * ns) : nullptr;
    double* dX = hst ? a.get<double>(B * ns * Tw) : X;
    if (!pass) { int rc = ensure_ws(h, a.off); if (rc) return rc; continue; }
    BootArgs ba{};
    int rc = stage_in(h, F0, dF0, (size_t)Tw * r, mem, &ba.F0); if (rc) return rc;
    rc = stage_in(h, resid, dre, (size_t)nres * r, mem, &ba.resid); if (rc) return rc;
    rc = stage_in(h, beta, dbe, (size_t)K * r, mem, &ba.beta); if (rc) return rc;
    rc = stage_in(h, lam, dla, (size_t)ns * r, mem, &ba.lam); if (rc) return rc;
    rc = stage_in(h, uar_coef, dac, (size_t)ns * Lg, mem, &ba.uar_coef); if (rc) return rc;
    rc = stage_in(h, uar_ser, dse, (size_t)ns, mem, &ba.uar_ser); if (rc) return rc;
    rc = stage_in(h, data, dda, (size_t)Tw * ns, mem, &ba.data); if (rc) return rc;
    ba.X = dX; ba.Tw = Tw; ba.ns = ns; ba.r = r; ba.p = p; ba.L = Lg; ba.nres = nres; ba.burn = o->burn; ba.seed = o->seed; ba.rep0 = o->rep0;
    DFM_SET_SMEM(k_bootstrap_panels, smem);
    L(k_bootstrap_panels, batch, 1, 256, smem, ba);
    if (hst) { rc = copy_out(h, X, dX, B * ns * Tw, mem); if (rc) return rc; }
  }
  return finish(h, mem);
}

// One call for the whole C4 replication step (SURVEY.md 8b: "one panel + B bootstrap seeds"): resample -> standardise + PCA
// + ALS (estimate_factor!, :328-382) -> sign alignment -> factor VAR (:444-492) -> IRF (:793-825), device resident between
// the stages.  The stages are the public entry points above run on temporaries of this call.
int dfm_bootstrap_irf(dfm_handle* h, const dfm_boot_opts* o, const double* F0, const double* resid, const double* beta,
                      const double* lam, const double* uar_coef, const double* uar_ser, const double* data, int nt_min,
                      double tol, int H, double* irf, int* als_iters, int* als_status) {
  if (!h || !o || !F0 || !resid || !beta || !lam || !uar_coef || !uar_ser || !data || !irf || H <= 0)
    return fail(h, DFM_ERR_ARG, "dfm_bootstrap_irf: bad argument");
  const int Tw = o->T, ns = o->ns, r = o->r, p = o->p, Lg = o->n_uarlag, nres = o->n_resid, batch = o->batch, mem = o->mem;
  if (Tw <= p || ns <= 0 || r <= 0 || p <= 0 || Lg <= 0 || nres <= 0 || batch <= 0) return fail(h, DFM_ERR_ARG, "dfm_bootstrap_irf: bad shape");
  CK(cudaSetDevice(h->device));
  const size_t B = batch; const int k = r * p, K = 1 + k;
  // temporaries of this call (the stages' own scratch lives in the handle's workspace)
  const size_t nin[7] = {(size_t)Tw * r, (size_t)nres * r, (size_t)K * r, (size_t)ns * r, (size_t)ns * Lg, (size_t)ns, (size_t)Tw * ns};
  const double* hin[7] = {F0, resid, beta, lam, uar_coef, uar_ser, data};
  size_t tot = 0, off[16];
  auto take = [&](size_t n) { size_t o_ = tot; tot += (n * 8 + 255) & ~(size_t)255; return o_; };
  for (int i = 0; i < 7; ++i) off[i] = take(nin[i]);
  const size_t oX = take(B * ns * Tw), oF = take(B * Tw * r), oM = take(B * k * k), oQ = take(B * r * k), oG = take(B * k * r),
               oI = take(B * (size_t)r * H * r);
  char* base = nullptr;
  CK(cudaMalloc((void**)&base, tot));
  auto D = [&](size_t o_) { return reinterpret_cast<double*>(base + o_); };
#define BI_FAIL(rc_) do { int r__ = (rc_); if (r__) { cudaStreamSynchronize(h->stream); cudaFree(base); return r__; } } while (0)
  const double* din[7];
  for (int i = 0; i < 7; ++i) {
    if (mem == DFM_MEM_HOST) {
      if (cudaMemcpyAsync(D(off[i]), hin[i], nin[i] * 8, cudaMemcpyHostToDevice, h->stream) != cudaSuccess) BI_FAIL(fail(h, DFM_ERR_CUDA, "dfm_bootstrap_irf: upload failed"));
      din[i] = D(off[i]);
    } else din[i] = hin[i];
  }
  dfm_boot_opts ob = *o; ob.mem = DFM_MEM_DEVICE;
  BI_FAIL(dfm_bootstrap_panels(h, &ob, din[0], din[1], din[2], din[3], din[4], din[5], din[6], D(oX)));
  dfm_factor_opts fo{}; fo.T = Tw; fo.N = ns; fo.r = r; fo.nt_min = nt_min; fo.tol = tol; fo.max_iter = 100000000; fo.compute_r2 = 0;
  fo.n_constr = 0; fo.batch = batch; fo.mem = DFM_MEM_DEVICE;
  std::vector<dfm_factor_stats> fs(B);
  BI_FAIL(dfm_estimate_factor(h, D(oX), &fo, nullptr, D(oF), nullptr, nullptr, nullptr, nullptr, fs.data()));
  for (size_t b = 0; b < B; ++b) { if (als_iters) als_iters[b] = fs[b].iters; if (als_status) als_status[b] = fs[b].status; }
  L(k_sign_align, batch, 1, 128, 48 * 8, D(oF), din[0], Tw, r);
  int rc = dfm_estimate_var(h, D(oF), Tw, r, p, 1, batch, DFM_MEM_DEVICE, nullptr, nullptr, nullptr, D(oM), D(oQ), D(oG));
  if (rc != DFM_OK && rc != DFM_ERR_NOT_PD && rc != DFM_ERR_TOO_FEW_OBS) BI_FAIL(rc);       // (all panels failed: records stay NaN)
  std::vector<int> ids(r); for (int j = 0; j < r; ++j) ids[j] = j;
  double* dI = mem == DFM_MEM_HOST ? D(oI) : irf;
  BI_FAIL(dfm_irf(h, D(oM), D(oQ), D(oG), k, r, H, r, ids.data(), batch, DFM_MEM_DEVICE, dI));
  if (mem == DFM_MEM_HOST && cudaMemcpyAsync(irf, dI, B * (size_t)r * H * r * 8, cudaMemcpyDeviceToHost, h->stream) != cudaSuccess)
    BI_FAIL(fail(h, DFM_ERR_CUDA, "dfm_bootstrap_irf: download failed"));
  cudaError_t e = cudaStreamSynchronize(h->stream);
  cudaFree(base);
#undef BI_FAIL
  CK(e);
  return DFM_OK;
}

// ------------------------------------------------------------------------------------ (f)3: percentile bands
// ------------------------------------------------------------------------------------ f4: instability tests
int dfm_instability(dfm_handle* h, const double* data, const double* F, int T, int ns, int r, int q, int T_break, double ccut,
                    int min_obs, int mem, double* chow, double* qlr, double* qlr0, int* status) {
  if (!h || !data || !F || !chow || !qlr || T <= 2 || ns <= 0 || r <= 0 || r > 16 || q < 0 || q > 7 || T_break <= 0 || T_break >= T ||
      !(ccut > 0.0 && ccut < 0.5) || min_obs < 0)
    return fail(h, DFM_ERR_ARG, "dfm_instability: bad argument (r <= 16, q <= 7, 0 < ccut < 0.5)");
  const size_t smem = inst_smem_doubles(T, r) * 8;
  if (smem > kMaxSmem) return fail(h, DFM_ERR_UNSUPPORTED, "dfm_instability: T x r too large for one CTA per series");
  CK(cudaSetDevice(h->device));
  for (int pass = 0; pass < 2; ++pass) {
    Arena a(pass ? h->ws : nullptr);
    double* dD = mem == DFM_MEM_HOST ? a.get<double>((size_t)T * ns) : nullptr;
    double* dF = mem == DFM_MEM_HOST ? a.get<double>((size_t)T * r) : nullptr;
    double* dc = a.get<double>(ns); double* dq = a.get<double>(ns); double* dq0 = a.get<double>(ns); int* dst = a.get<int>(ns);
    if (!pass) { int rc = ensure_ws(h, a.off); if (rc) return rc; continue; }
    const double *x, *f;
    int rc = stage_in(h, data, dD, (size_t)T * ns, mem, &x); if (rc) return rc;
    rc = stage_in(h, F, dF, (size_t)T * r, mem, &f); if (rc) return rc;
    CK(cudaMemsetAsync(dst, 0, ns * sizeof(int), h->stream));
    DFM_SET_SMEM(k_instability, smem);
    L(k_instability, ns, 1, 256, smem, x, f, T, ns, r, q, T_break, ccut, min_obs, dc, dq, qlr0 ? dq0 : (double*)nullptr, dst);
    rc = copy_out(h, chow, dc, ns, mem); if (rc) return rc;
    rc = copy_out(h, qlr, dq, ns, mem); if (rc) return rc;
    if (qlr0) { rc = copy_out(h, qlr0, dq0, ns, mem); if (rc) return rc; }
    if (status) { rc = copy_out(h, status, dst, ns, mem); if (rc) return rc; }
  }
  return finish(h, mem);
}

int dfm_fit_correlation(dfm_handle* h, const double* data, const double* F, const double* F_alt, int T, int ns, int r, int T_break,
                        int min_obs, int mem, double* cor, int* status) {
  if (!h || !data || !F || !F_alt || !cor || T <= 2 || ns <= 0 || r <= 0 || r > 48 || T_break <= 0 || T_break >= T || min_obs < 0)
    return fail(h, DFM_ERR_ARG, "dfm_fit_correlation: bad argument");
  CK(cudaSetDevice(h->device));
  for (int pass = 0; pass < 2; ++pass) {
    Arena a(pass ? h->ws : nullptr);
    double* dD = mem == DFM_MEM_HOST ? a.get<double>((size_t)T * ns) : nullptr;
    double* dF = mem == DFM_MEM_HOST ? a.get<double>((size_t)T * r) : nullptr;
    double* dFa = mem == DFM_MEM_HOST ? a.get<double>((size_t)T * r) : nullptr;
    double* dc = a.get<double>(ns); int* dst = a.get<int>(ns);
    if (!pass) { int rc = ensure_ws(h, a.off); if (rc) return rc; continue; }
    const double *x, *f, *fa;
    int rc = stage_in(h, data, dD, (size_t)T * ns, mem, &x); if (rc) return rc;
    rc = stage_in(h, F, dF, (size_t)T * r, mem, &f); if (rc) return rc;
    rc = stage_in(h, F_alt, dFa, (size_t)T * r, mem, &fa); if (rc) return rc;
    CK(cudaMemsetAsync(dst, 0, ns * sizeof(int), h->stream));
    L(k_fit_corr, ns, 1, 128, (size_t)(2 * (r * r + 2 * r) + 64 + 48 + 8) * 8, x, f, fa, T, ns, r, T_break, min_obs, dc, dst);
    rc = copy_out(h, cor, dc, ns, mem); if (rc) return rc;
    if (status) { rc = copy_out(h, status, dst, ns, mem); if (rc) return rc; }
  }
  return finish(h, mem);
}

int dfm_percentiles(dfm_handle* h, const double* recs, long long n, int d, const double* q, int nq, int mem, double* out) {
  if (!h || !recs || !q || !out || n <= 0 || d <= 0 || nq <= 0 || nq > 64) return fail(h, DFM_ERR_ARG, "dfm_percentiles: bad argument");
  for (int k = 0; k < nq; ++k) if (!(q[k] >= 0.0 && q[k] <= 100.0)) return fail(h, DFM_ERR_ARG, "dfm_percentiles: q outside [0, 100]");
  long long npad = 2; while (npad < n) npad <<= 1;
  size_t smem = (size_t)(npad + 2) * 8;
  if (smem > kMaxSmem) return fail(h, DFM_ERR_UNSUPPORTED, "dfm_percentiles: more than 16384 replications");
  CK(cudaSetDevice(h->device));
  for (int pass = 0; pass < 2; ++pass) {
    Arena a(pass ? h->ws : nullptr);
    double* dr = mem == DFM_MEM_HOST ? a.get<double>((size_t)n * d) : nullptr;
    double* dq = a.get<double>(nq); double* dout = mem == DFM_MEM_HOST ? a.get<double>((size_t)nq * d) : out;
    if (!pass) { int rc = ensure_ws(h, a.off); if (rc) return rc; continue; }
    const double* r_; int rc = stage_in(h, recs, dr, (size_t)n * d, mem, &r_); if (rc) return rc;
    CK(cudaMemcpyAsync(dq, q, nq * sizeof(double), cudaMemcpyHostToDevice, h->stream));      // q is always a host array
    DFM_SET_SMEM(k_percentiles, smem);
    L(k_percentiles, d, 1, 256, smem, r_, (int)n, d, dq, nq, (int)npad, dout);
    if (mem == DFM_MEM_HOST) { rc = copy_out(h, out, dout, (size_t)nq * d, mem); if (rc) return rc; }
    else CK(cudaStreamSynchronize(h->stream));                                               // (dq lives in the shared workspace)
  }
  return finish(h, mem);
}

int dfm_allgather_results(dfm_handle* h, void* nccl_comm, const double* send, double* recv, long long count) {
  if (!h || !nccl_comm || !send || !recv || count <= 0) return fail(h, DFM_ERR_ARG, "dfm_allgather_results: bad argument");
#ifdef DFM_EMU
  return DFM_ERR_NCCL;
#else
  typedef int (*allgather_fn)(const void*, void*, size_t, int, void*, cudaStream_t);
  static allgather_fn fn = nullptr;
  if (!fn) {
    // the communicator was created by the NCCL the caller already loaded (NCCL.jl, torch's bundled copy, ...): use THAT
    // library's ncclAllGather when it is visible in the process, and only otherwise load one by name
    fn = (allgather_fn)dlsym(RTLD_DEFAULT, "ncclAllGather");
    if (!fn) {
      const char* names[] = {"libnccl.so.2", "libnccl.so"};
      void* lib = nullptr;
      for (const char* n : names) { lib = dlopen(n, RTLD_NOW | RTLD_GLOBAL); if (lib) break; }
      if (!lib) return fail(h, DFM_ERR_NCCL, "libnccl not found");
      fn = (allgather_fn)dlsym(lib, "ncclAllGather");
    }
    if (!fn) return fail(h, DFM_ERR_NCCL, "ncclAllGather not found");
  }
  CK(cudaSetDevice(h->device));
  const int kNcclFloat64 = 8;      // ncclDataType_t: ncclFloat64 = ncclDouble = 8 in every NCCL 2.x release (nccl.h)
  int rc = fn(send, recv, (size_t)count, kNcclFloat64, nccl_comm, h->stream);
  if (rc != 0) return fail(h, DFM_ERR_NCCL, "ncclAllGather failed");
  return DFM_OK;
#endif
}

}  // extern "C"
