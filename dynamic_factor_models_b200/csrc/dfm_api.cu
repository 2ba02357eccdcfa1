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
#include "dfm_kernels_ssb.cuh"
#include "dfm_kernels_gibbs.cuh"
#include "dfm_kernels_resp.cuh"
#include "dfm_kernels_hd.cuh"
#include "dfm_kernels_sign.cuh"
#include "dfm_kernels_narr.cuh"
#include "dfm_kernels_proxy.cuh"
#include <algorithm>
#include <cmath>
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
  size_t attr = 48 * 1024;                                    // the attribute's default; a set value replaces it, up or down
  {
    std::lock_guard<std::mutex> lk(g_emu_attr_mu);
    auto it = g_emu_smem_attr.find(kern);
    if (it != g_emu_smem_attr.end()) attr = it->second;
  }
  const bool ok = smem <= attr && nt >= 1 && nt <= 1024 && gx >= 1 && gx <= 2147483647LL && gy >= 1 &&
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
  char* rws;                   // second workspace: temporaries of entry points that call other entry points (which use ws and
  size_t rws_bytes;            //   may regrow it), kept across calls like ws
  long long launches;
  int profile;                 // 1: bracket every kernel launch with CUDA events (dfm_profile_*)
  std::vector<ProfRec>* prof;
  char err[256];
};

namespace {

const size_t kMaxSmem = 220 * 1024;
// Entry points whose launches put the batch on gridDim.y (at most 65535 blocks) refuse larger batches with
// DFM_ERR_UNSUPPORTED; callers split such batches.
const int kMaxGridBatch = 65535;
const int kReadyChunk = 32;                                    // panels per upload chunk of the streaming host path
const int kMaxReadyChunks = (kMaxGridBatch + kReadyChunk - 1) / kReadyChunk;   // "landed" flags of the largest batch

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

// the second workspace (dfm_handle::rws), grown as ensure_ws grows ws
int ensure_rws(dfm_handle* h, size_t bytes) {
  if (bytes <= h->rws_bytes) return DFM_OK;
  if (h->rws) { CK(cudaStreamSynchronize(h->stream)); CK(cudaFree(h->rws)); h->rws = nullptr; h->rws_bytes = 0; }
  void* p = nullptr;
  CK(cudaMalloc(&p, bytes));
  h->rws = (char*)p; h->rws_bytes = bytes;
  return DFM_OK;
}

// Lays out a call's device buffers: layout(a) walks them once on a null Arena to size them, the workspace grows to that size,
// and layout(a) walks them again to place them.  in_rws: the second workspace (dfm_handle::rws), for the temporaries of entry
// points that call other entry points.
template <class Lay> int lay_out(dfm_handle* h, Lay&& layout, bool in_rws = false) {
  Arena probe(nullptr);
  layout(probe);
  int rc = in_rws ? ensure_rws(h, probe.off) : ensure_ws(h, probe.off);
  if (rc) return rc;
  Arena a(in_rws ? h->rws : h->ws);
  layout(a);
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

// One output of an entry point: dst, the caller's array of `per` elements a row (a panel, a model, a draw; nullptr: not asked
// for).  The kernels write buf when there is one, else dst in place; flush copies the rows they wrote to dst.
template <typename T> struct OutSlot {
  T* dst = nullptr;
  T* buf = nullptr;
  size_t per = 0;
  // where the kernels write the rows that start at row j0 (nullptr: nowhere)
  T* at(long long j0) const { return buf ? buf : dst ? dst + j0 * per : nullptr; }
  int flush(dfm_handle* h, long long j0, long long n, int mem) const {
    return copy_out(h, dst ? dst + j0 * per : nullptr, at(j0), n * per, mem);
  }
};

// an output the kernels write only when it is asked for: in place in device memory, through a staging buffer of B rows to host
// memory
template <typename T> OutSlot<T> staged(Arena& a, T* dst, size_t per, size_t B, bool hst) {
  return {dst, hst && dst ? a.get<T>(B * per) : nullptr, per};
}

// an output the kernels write whether or not it is asked for: in place when it is asked for in device memory, else into the
// buffer (allocated either way, so that the layout's size does not depend on dst)
template <typename T> OutSlot<T> scratch(Arena& a, T* dst, size_t per, size_t B, bool hst) {
  T* buf = a.get<T>(B * per);
  return {dst, hst || !dst ? buf : nullptr, per};
}

// the copy-back of the n rows from j0 of every slot, up to the first error
template <typename... T> int flush(dfm_handle* h, long long j0, long long n, int mem, const OutSlot<T>&... s) {
  int rc = DFM_OK;
  ((rc = rc ? rc : s.flush(h, j0, n, mem)), ...);
  return rc;
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

// any NaN in the panel / parameters?  (the fused path handles balanced panels only)  Lam == nullptr: the panel only.
namespace dfm {
__global__ void k_em_scan_fused(const double* __restrict__ X, const double* __restrict__ Lam, const double* __restrict__ R,
                                int T, int N, int r, int* flag) {
  int i = DFM_BX, b = DFM_BY;
  const double* x = X + ((size_t)b * N + i) * T;
  int bad = 0;
  for (int t = DFM_TID; t < T; t += DFM_NT) if (is_nan(x[t])) bad = 1;
  if (Lam && DFM_TID == 0) { for (int a = 0; a < r; ++a) if (is_nan(Lam[(size_t)b * N * r + i + (size_t)N * a])) bad = 1; if (is_nan(R[(size_t)b * N + i])) bad = 1; }
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

// Turn window of the `grid` CTAs of a TMA kernel (f2_produce): F2_L2WIN_PCT of L2 split over the CTAs active in a round,
// in copies per pass turn; win[0] for the full rounds, win[1] for the tail round.
static void l2_turn_plan(const dfm_handle* h, int grid, int B, int N, int win[2]) {
  const long long copy = 64LL * F2_SBS * F2_TC, nsg = (N + 8 * F2_SBS - 1) / (8 * F2_SBS);   // bytes of one copy, groups per panel
  const int tail = (B % grid) ? B % grid : grid;
  win[0] = (int)std::min(nsg, (long long)h->l2_bytes * F2_L2WIN_PCT / 100 / (grid * copy));
  win[1] = (int)std::min(nsg, (long long)h->l2_bytes * F2_L2WIN_PCT / 100 / (tail * copy));
}

// One launch of the fused EM kernel over all panels of fa (fa.scratch: min(B, nsm * 8) * T * FUSED_SCR(r) doubles):
// k_em_fused2 (TMA panel ring, even T) when use2, else k_em_fused.
static int launch_em_fused(dfm_handle* h, FusedArgs fa, int r, bool use2) {
  return dispatch<1, 8>(r, [&](auto R) -> int {
    constexpr int RT = decltype(R)::value;
    if (use2) {
      const size_t smem = fused2_smem_doubles<RT>(fa.T, fa.N) * 8;
      const int grid = resident_grid(h, k_em_fused2<RT>, 256, smem, fa.B);
      l2_turn_plan(h, grid, fa.B, fa.N, fa.l2_win);
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
// cs.off != nullptr (restrictions on the loadings): k_emb_mstep_constr with its scratch for the correction.
static void emb_launch_M(dfm_handle* h, const EmbPlan& e, const double* x, const double* dFs, const double* dSff, int T, int N, int r, int batch,
                         double* dL, double* dR, double* dW, double* dlogR, EmState* st, EmConstr cs = EmConstr{}) {
  dispatch<1, 4>(e.ncb, [&](auto C) {
    constexpr int NCB = decltype(C)::value;
    if (cs.off) {
      const size_t sm = e.smM + (size_t)em_constr_scratch(r) * 8;
      DFM_SET_SMEM(k_emb_mstep_constr<NCB>, sm);
      L(k_emb_mstep_constr<NCB>, e.ntM, e.tsM * batch, 256, sm, x, dFs, dSff, T, N, r, e.tsM, e.tper, batch, e.Spart, e.sxxpart,
        e.counters + (size_t)batch * e.ntE, dL, dR, dW, dlogR, e.Cpart, st, cs);
      return;
    }
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

// General multi-kernel EM path on device-resident data (any r, p, missing data).  cs: restrictions on the loadings (the
// device CSR of em_kalman_impl; off == nullptr: none), applied by the two measurement M-step kernels.
static int run_em_general(dfm_handle* h, const double* x, const dfm_em_opts* o, const EmBufs& d, const GenBufs& g, int want_psf,
                          EmConstr cs) {
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
  // k_em_mstep_series' shared memory is set on every call: a call with restrictions sets a size for its r, and the
  // attribute (per kernel, per process) would otherwise cap the launches of later calls at a larger r
  const size_t smS = (size_t)(2 * np + r + 8 + (cs.off ? em_constr_scratch(r) : 0)) * 8;
  if (any_missing || !emb.on) DFM_SET_SMEM(k_em_mstep_series, smS);
  int h_active = batch;
  for (int it = 0; it < mi && h_active > 0; ++it) {
    if (any_missing) L(k_em_contract, nblkC, batch, ntC, ((size_t)(np + r) * ntC + 8) * 8, x, d.L, g.W, d.R, g.logR, g.C, T, N, r, g.Bt, g.qt, g.slr, g.nt, g.Ct, d.st);
    if (any_bal) {                                                          // (each returns at once for panels of the other kind)
      if (!emb.on) L(k_em_contract_bal, (T + 31) / 32, batch, 256, 8 * 32 * 3 * 8, x, g.W, d.R, g.logR, T, N, r, g.Bt, g.qt, g.slr, g.nt, d.st);
      else emb_launch_E(h, emb, x, g.W, d.R, g.logR, T, N, r, batch, g.Bt, g.qt, g.slr, g.nt, d.st);
    }
    launch_filter_smooth(h, ncl, g, batch, T, r, p, d.A, d.Q, d.P0, d.Fs, d.PsF, d.ll, d.st, mi, o->tol, want_psf);
    if (any_missing || !emb.on) {
      L(k_em_mstep_series, N, batch, 64, smS, x, d.Fs, d.PsF, g.Sff, T, N, r, d.L, d.R, d.st, emb_on, cs);
    }
    if (any_bal && emb.on) {
      emb_launch_M(h, emb, x, d.Fs, g.Sff, T, N, r, batch, d.L, d.R, g.W, g.logR, d.st, cs);
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
    l2_turn_plan(h, grid, fa.B, fa.N, fa.l2_win);
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
  const int chunk = kReadyChunk;                               // ~25 MB of C2-shaped panels: the first CTAs start early
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
    // The question is whether the CALLER passed a NaN (a missing cell; a series out of the model), as in the scan the
    // other host path runs before the kernel.  d.L / d.R hold what the kernel wrote by now, and a panel that failed
    // numerically on clean data leaves NaNs there: scanning them would send the whole batch through the general path
    // for one bad panel.  So: the caller's Lam and R on the host, X on the device.
    bool nan_in = false;
    for (size_t e = 0; e < B * N * r && !nan_in; ++e) nan_in = std::isnan(init->Lam[e]);
    for (size_t e = 0; e < B * N && !nan_in; ++e) nan_in = std::isnan(init->R[e]);
    if (!nan_in) {
      CK(cudaMemsetAsync(d.flag, 0, sizeof(int), h->stream));
      L(k_em_scan_fused, N, batch, 64, 0, d.X, (const double*)nullptr, (const double*)nullptr, T, N, r, d.flag);
      int hflag = 0;
      CK(cudaMemcpyAsync(&hflag, d.flag, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
      CK(cudaStreamSynchronize(h->stream));
      nan_in = hflag != 0;
    }
    *fallback = nan_in;
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
  if (h->rws) cudaFree(h->rws);
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
  h->device = device; h->ws = nullptr; h->ws_bytes = 0; h->rws = nullptr; h->rws_bytes = 0; h->launches = 0; h->err[0] = 0;
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
  const bool hst = mem == DFM_MEM_HOST;
  double *dX, *dm, *ds;
  OutSlot<double> oXs;
  int rc = lay_out(h, [&](Arena& a) {
    dX = hst ? a.get<double>(B * TN) : nullptr;
    oXs = staged(a, Xs, TN, B, hst);
    dm = a.get<double>(B * N); ds = a.get<double>(B * N);
  });
  if (rc) return rc;
  const double* x; rc = stage_in(h, X, dX, B * TN, mem, &x); if (rc) return rc;
  L(k_standardize, N, batch, 128, 48 * 8, x, T, N, oXs.at(0), dm, ds, (double*)nullptr, (int*)nullptr);
  rc = oXs.flush(h, 0, B, mem); if (rc) return rc;
  rc = copy_out(h, xmean, dm, B * N, mem); if (rc) return rc;
  rc = copy_out(h, xstd, ds, B * N, mem); if (rc) return rc;
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
  const bool hst = mem == DFM_MEM_HOST;
  double *dX, *G, *V, *Ysub;
  int *bal, *nbal, *status;
  OutSlot<double> oF;
  int rc = lay_out(h, [&](Arena& a) {
    dX = hst ? a.get<double>(B * TN) : nullptr;
    oF = staged(a, score, (size_t)T * r, B, hst);
    bal = a.get<int>(B * N); nbal = a.get<int>(B); status = a.get<int>(B);
    G = a.get<double>(B * nmax * nmax); V = a.get<double>(B * nmax * nmax);
    Ysub = a.get<double>(B * nmax * PCA_MMAX);
  });
  if (rc) return rc;
  const double* x; rc = stage_in(h, X, dX, B * TN, mem, &x); if (rc) return rc;
  CK(cudaMemsetAsync(status, 0, B * sizeof(int), h->stream));
  rc = run_pca(h, x, T, N, r, batch, nullptr, bal, nbal, G, V, Ysub, oF.at(0), status, nullptr); if (rc) return rc;
  rc = oF.flush(h, 0, B, mem); if (rc) return rc;
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
  double *dX, *dXs, *dm, *ds, *css, *G, *V, *Ysub, *dF, *dLam, *dR2, *FtF, *LtL, *ssrp, *cR, *cr, *gsys;
  int *cn, *bal, *nbal, *active, *cidx;
  AlsState* st;
  int rc = lay_out(h, [&](Arena& a) {
    dX = mem == DFM_MEM_HOST ? a.get<double>(B * TN) : nullptr;
    dXs = a.get<double>(B * TN);
    dm = a.get<double>(B * N); ds = a.get<double>(B * N); css = a.get<double>(B * N);
    cn = a.get<int>(B * N); st = a.get<AlsState>(B);
    bal = a.get<int>(B * N); nbal = a.get<int>(B); active = a.get<int>(4);
    G = F_init ? nullptr : a.get<double>(B * nmax * nmax); V = F_init ? nullptr : a.get<double>(B * nmax * nmax);
    Ysub = F_init ? nullptr : a.get<double>(B * nmax * PCA_MMAX);
    dF = a.get<double>(B * T * r); dLam = a.get<double>(B * N * r); dR2 = a.get<double>(B * N);
    FtF = a.get<double>(B * r * r); LtL = a.get<double>(B * r * r); ssrp = a.get<double>(B * nblk);
    cidx = a.get<int>(nc + 1); cR = a.get<double>((size_t)nc * r + 1); cr = a.get<double>(nc + 1);
    gsys = sys_global ? a.get<double>(B * nblk * (size_t)(np + r) * ntF) : nullptr;
  });
  if (rc) return rc;
  const double* x; rc = stage_in(h, X, dX, B * TN, mem, &x); if (rc) return rc;
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
  const bool hst = mem == DFM_MEM_HOST;
  double *dD, *dFb, *dl, *dr2, *dac, *dser, *scr, *dcon, *cR, *cr;
  int *status, *cidx;
  OutSlot<double> oRes;
  int rc = lay_out(h, [&](Arena& a) {
    dD = hst ? a.get<double>(B * T * ns) : nullptr;
    dFb = hst ? a.get<double>(B * T * r) : nullptr;
    dl = a.get<double>(B * ns * r); dr2 = a.get<double>(B * ns);
    dac = a.get<double>(B * ns * L_); dser = a.get<double>(B * ns);
    scr = a.get<double>(B * ns * T); status = a.get<int>(B);
    dcon = constant ? a.get<double>(B * ns) : nullptr;
    oRes = staged(a, resid, (size_t)ns * T, B, hst);
    cidx = a.get<int>(nc + 1); cR = a.get<double>((size_t)nc * r + 1); cr = a.get<double>(nc + 1);
  });
  if (rc) return rc;
  const double* d; const double* f;
  rc = stage_in(h, data, dD, B * T * ns, mem, &d); if (rc) return rc;
  rc = stage_in(h, F, dFb, B * T * r, mem, &f); if (rc) return rc;
  if (nc > 0) {
    CK(cudaMemcpyAsync(cidx, o->constr_index, nc * sizeof(int), cudaMemcpyHostToDevice, h->stream));
    CK(cudaMemcpyAsync(cR, o->constr_R, (size_t)nc * r * sizeof(double), cudaMemcpyHostToDevice, h->stream));
    CK(cudaMemcpyAsync(cr, o->constr_r, nc * sizeof(double), cudaMemcpyHostToDevice, h->stream));
  }
  CK(cudaMemsetAsync(status, 0, B * sizeof(int), h->stream));
  size_t wk = std::max<size_t>((size_t)K * nc + (size_t)nc * (nc + 1) / 2 + nc, (size_t)L_ * (L_ + 1) / 2 + L_);
  size_t sm = (size_t)(np + K + 8 + wk) * 8;
  L(k_loading, ns, batch, 64, sm, d, f, T, ns, r, o->nt_min, L_, dl, dr2, dac, dser, scr, nc, cidx, cR, cr, status, dcon, oRes.at(0));
  rc = copy_out(h, lambda, dl, B * ns * r, mem); if (rc) return rc;
  rc = copy_out(h, r2, dr2, B * ns, mem); if (rc) return rc;
  rc = copy_out(h, uar_coef, dac, B * ns * L_, mem); if (rc) return rc;
  rc = copy_out(h, uar_ser, dser, B * ns, mem); if (rc) return rc;
  if (constant) { rc = copy_out(h, constant, dcon, B * ns, mem); if (rc) return rc; }
  rc = oRes.flush(h, 0, B, mem); if (rc) return rc;
  if (status_out) {
    // per-panel status (0, or DFM_ERR_NOT_PD when a regression / constraint / AR step of some series was singular;
    // the affected series carry NaN).  Always a HOST array.
    CK(cudaMemcpyAsync(status_out, status, B * sizeof(int), cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
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
  double *dFb, *db, *dres, *dse, *dM, *dQ, *dG;
  int* status;
  int rc = lay_out(h, [&](Arena& a) {
    dFb = mem == DFM_MEM_HOST ? a.get<double>(B * T * r) : nullptr;
    db = a.get<double>(B * K * r); dres = a.get<double>(B * T * r); dse = a.get<double>(B * r * r);
    dM = a.get<double>(B * k * k); dQ = a.get<double>(B * r * k); dG = a.get<double>(B * k * r);
    status = a.get<int>(B);
  });
  if (rc) return rc;
  const double* f; rc = stage_in(h, F, dFb, B * T * r, mem, &f); if (rc) return rc;
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
  return finish(h, mem);
}

// ------------------------------------------------------------------------------------ a11
int dfm_irf(dfm_handle* h, const double* M, const double* Q, const double* G, int k, int r, int H, int n_shock,
            const int* shock_ids, int batch, int mem, double* irf) {
  if (!h || !M || !Q || !G || !shock_ids || !irf || k <= 0 || r <= 0 || H <= 0 || n_shock <= 0 || batch <= 0)
    return fail(h, DFM_ERR_ARG, "dfm_irf: bad argument");
  for (int j = 0; j < n_shock; ++j) if (shock_ids[j] < 0 || shock_ids[j] >= r) return fail(h, DFM_ERR_ARG, "dfm_irf: shock id out of range");
  if (batch > kMaxGridBatch) return fail(h, DFM_ERR_UNSUPPORTED, "dfm_irf: batch > 65535");
  const size_t smI = irf_smem_doubles(k) * 8;
  if (smI > kMaxSmem) return fail(h, DFM_ERR_UNSUPPORTED, "dfm_irf: state dimension k too large (k > 14076)");
  CK(cudaSetDevice(h->device));
  size_t B = batch;
  const bool hst = mem == DFM_MEM_HOST;
  double *dM, *dQ, *dG;
  int* ids;
  OutSlot<double> oI;
  int rc = lay_out(h, [&](Arena& a) {
    dM = hst ? a.get<double>(B * k * k) : nullptr;
    dQ = hst ? a.get<double>(B * r * k) : nullptr;
    dG = hst ? a.get<double>(B * k * r) : nullptr;
    oI = staged(a, irf, (size_t)r * H * n_shock, B, hst);
    ids = a.get<int>(n_shock);
  });
  if (rc) return rc;
  const double *m, *q, *g;
  rc = stage_in(h, M, dM, B * k * k, mem, &m); if (rc) return rc;
  rc = stage_in(h, Q, dQ, B * r * k, mem, &q); if (rc) return rc;
  rc = stage_in(h, G, dG, B * k * r, mem, &g); if (rc) return rc;
  CK(cudaMemcpyAsync(ids, shock_ids, n_shock * sizeof(int), cudaMemcpyHostToDevice, h->stream));
  DFM_SET_SMEM(k_irf, smI);                                // (every call: a lower value from an earlier call may be in place)
  L(k_irf, n_shock, batch, 64, smI, m, q, g, k, r, H, n_shock, ids, oI.at(0));
  rc = oI.flush(h, 0, B, mem); if (rc) return rc;
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
  double *dX, *dFb, *dL, *dR, *dA, *dQ, *dres;
  int* status;
  EmState* est = nullptr; int* miss = nullptr; double *dFtF = nullptr, *dWs = nullptr, *dlogRs = nullptr;
  int rc = lay_out(h, [&](Arena& a) {
    dX = mem == DFM_MEM_HOST ? a.get<double>(B * TN) : nullptr;
    dFb = mem == DFM_MEM_HOST ? a.get<double>(B * T * r) : nullptr;
    dL = a.get<double>(B * N * r); dR = a.get<double>(B * N);
    dA = a.get<double>(B * r * k); dQ = a.get<double>(B * r * r); dres = a.get<double>(B * T * r);
    status = a.get<int>(B);
    if (embi.on) {
      est = a.get<EmState>(B); miss = a.get<int>(B); dFtF = a.get<double>(B * r * r); dWs = a.get<double>(B * N * r); dlogRs = a.get<double>(B * N);
      embi.Spart = a.get<double>((size_t)embi.tsM * B * N * r); embi.sxxpart = a.get<double>((size_t)embi.tsM * B * N);
      embi.Cpart = a.get<double>(B * embi.ntM * r * r); embi.counters = a.get<int>(B * (size_t)(embi.ntE + embi.ntM));
    }
  });
  if (rc) return rc;
  const double *x, *f;
  rc = stage_in(h, Xs, dX, B * TN, mem, &x); if (rc) return rc;
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
  return finish(h, mem);
}

// ------------------------------------------------------------------------------------ a'
// Restrictions on the loadings (dfm_lam_constr) as a host CSR grouped by series in their given order: offsets [N+1], rows
// [nc x r] row-major, values [nc].  `what`: the entry point, for the error messages.
struct ConstrCsr { int nc = 0; std::vector<int> off; std::vector<double> H, h; };

static int constr_csr(dfm_handle* h, const char* what, const dfm_lam_constr* con, int N, int r, ConstrCsr* cc) {
  char msg[160];
  auto bad = [&](const char* why) { snprintf(msg, sizeof(msg), "%s: %s", what, why); return fail(h, DFM_ERR_ARG, msg); };
  const int nc = con ? con->n_constr : 0;
  cc->nc = nc;
  if (nc < 0) return bad("n_constr < 0");
  if (nc == 0) return DFM_OK;
  if (!con->index || !con->H || !con->h) return bad("null restriction array");
  std::vector<int>& coff = cc->off;
  coff.assign((size_t)N + 1, 0);
  for (int q = 0; q < nc; ++q) {
    const int i = con->index[q];
    if (i < 0 || i >= N) return bad("restriction index outside [0, N)");
    if (!std::isfinite(con->h[q])) return bad("non-finite restriction value");
    for (int a = 0; a < r; ++a)
      if (!std::isfinite(con->H[q + (size_t)nc * a])) return bad("non-finite restriction row");
    if (++coff[i + 1] > r) return bad("more than r restriction rows on one series");
  }
  for (int i = 0; i < N; ++i) coff[i + 1] += coff[i];
  cc->H.resize((size_t)nc * r); cc->h.resize(nc);
  std::vector<int> fill(coff.begin(), coff.end() - 1);
  for (int q = 0; q < nc; ++q) {
    const int dst = fill[con->index[q]]++;
    for (int a = 0; a < r; ++a) cc->H[(size_t)dst * r + a] = con->H[q + (size_t)nc * a];
    cc->h[dst] = con->h[q];
  }
  return DFM_OK;
}

// The device copy of a CSR: cs's arrays from the arena (N + 1 ints, nc r and nc doubles); upload on the handle's stream.
static EmConstr constr_bufs(Arena& a, const ConstrCsr& cc, int N, int r) {
  EmConstr cs{};
  if (cc.nc) { cs.off = a.get<int>((size_t)N + 1); cs.H = a.get<double>((size_t)cc.nc * r); cs.h = a.get<double>(cc.nc); }
  return cs;
}

static int constr_upload(dfm_handle* h, const ConstrCsr& cc, const EmConstr& cs) {
  if (!cc.nc) return DFM_OK;              // (pageable sources: each copy returns once its source has been staged)
  CK(cudaMemcpyAsync((void*)cs.off, cc.off.data(), cc.off.size() * sizeof(int), cudaMemcpyHostToDevice, h->stream));
  CK(cudaMemcpyAsync((void*)cs.H, cc.H.data(), cc.H.size() * 8, cudaMemcpyHostToDevice, h->stream));
  CK(cudaMemcpyAsync((void*)cs.h, cc.h.data(), cc.h.size() * 8, cudaMemcpyHostToDevice, h->stream));
  return DFM_OK;
}

// dfm_em_kalman and dfm_em_kalman_constrained.  con == nullptr or con->n_constr == 0: the unrestricted EM (same dispatch, same
// bits).  Otherwise the restriction is checked, uploaded once as a per-series CSR (rows grouped by series in their given order)
// and the call runs the general path, whatever the shape.
static int em_kalman_impl(dfm_handle* h, const double* X, const dfm_em_opts* o, const dfm_em_init* init, const dfm_lam_constr* con,
                          const dfm_em_out* out) {
  if (!h || !X || !o || !init || !out || !init->Lam || !init->R || !init->A || !init->Q)
    return fail(h, DFM_ERR_ARG, "dfm_em_kalman: null argument");
  int T = o->T, N = o->N, r = o->r, p = o->p, batch = o->batch, mem = o->mem, mi = o->max_iter;
  if (T <= 1 || N <= 0 || r <= 0 || r > 64 || p <= 0 || batch <= 0 || mi <= 0 || o->tol < 0)
    return fail(h, DFM_ERR_ARG, "dfm_em_kalman: bad shape/options");
  ConstrCsr cc;
  { int rc = constr_csr(h, "dfm_em_kalman_constrained", con, N, r, &cc); if (rc) return rc; }
  const int nc = cc.nc;
  if (nc > 0) {
    if (o->path == 2 || o->path == 3) return fail(h, DFM_ERR_UNSUPPORTED, "dfm_em_kalman_constrained: the fused paths take no restrictions");
  }
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
  const bool try_fused = (fused_ok || fused2_ok) && o->path != 1 && nc == 0;      // the path is only chosen after the NaN scan
  const bool use2 = fused2_ok && (o->path == 0 || o->path == 3) && nc == 0;
  const EmbPlan emb = emb_plan(T, N, r, batch, h->nsm);
  EmBufs d;
  GenBufs g;
  EmConstr cs;
  int rc = lay_out(h, [&](Arena& a) {
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
    g = gen_bufs(a, emb, B, T, N, r, p);        // also the fallback when the scan finds missing data
    cs = constr_bufs(a, cc, N, r);
  });
  if (rc) return rc;
  rc = constr_upload(h, cc, cs);
  if (rc) return rc;
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
  else rc = run_em_general(h, x, o, d, g, out->PF ? 1 : 0, cs);
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
  return finish(h, mem);
}

int dfm_em_kalman(dfm_handle* h, const double* X, const dfm_em_opts* o, const dfm_em_init* init, const dfm_em_out* out) {
  return em_kalman_impl(h, X, o, init, nullptr, out);
}

int dfm_em_kalman_constrained(dfm_handle* h, const double* X, const dfm_em_opts* o, const dfm_em_init* init, const dfm_lam_constr* constr,
                              const dfm_em_out* out) {
  return em_kalman_impl(h, X, o, init, constr, out);
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
  const bool hst = mem == DFM_MEM_HOST;
  SsStage s;
  OutSlot<double> oPF, oCom, oXh, oXv;
  rc = lay_out(h, [&](Arena& a) {
    s = ss_bufs(a, mem, H, B, Tp, N, r, p);
    oPF = staged(a, out->PF, (size_t)Tp * rr, B, hst);
    oCom = staged(a, out->common, TN, B, hst);
    oXh = staged(a, out->xhat, TN, B, hst);
    oXv = staged(a, out->xvar, TN, B, hst);
  });
  if (rc) return rc;
  rc = ss_estep(h, s, X, params, T, N, r, p, H, batch, mem);
  if (rc) return rc;
  L(k_ss_nan_failed, batch, 1, 256, 0, (const EmState*)s.st, Tp, r, s.Fs, s.PsF, s.ll);
  // ---- projection onto the series
  if (out->common || out->xhat || out->xvar) {
    DFM_SET_SMEM(k_ss_project, smP);
    const int nst = (N + SS_NS - 1) / SS_NS, ntt = (Tp + SS_TP - 1) / SS_TP;
    const int per = std::max(1, 65535 / nst);            // panels per launch (grid.y limit)
    for (int b0 = 0; b0 < batch; b0 += per) {
      const int nb = std::min(per, batch - b0);
      L(k_ss_project, ntt, nst * nb, 256, smP, s.x, (const double*)s.Fs, (const double*)s.PsF, s.pL, s.pR, (const EmState*)s.st, Tp, N, r,
        b0, oCom.at(0), oXh.at(0), oXv.at(0));
    }
  }
  // ---- results
  rc = copy_out(h, out->F, s.Fs, B * Tp * r, mem); if (rc) return rc;
  if (out->PF) {
    long long n = (long long)Tp * rr;
    L(k_unpack_psf, (int)std::min<long long>((n + 255) / 256, 1024), batch, 256, 0, s.PsF, Tp, r, oPF.at(0));
  }
  rc = flush(h, 0, B, mem, oPF, oCom, oXh, oXv); if (rc) return rc;
  rc = copy_out(h, out->loglik, s.ll, B, mem); if (rc) return rc;
  rc = copy_out(h, out->status, s.stat, B, mem); if (rc) return rc;
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
  const bool hst = mem == DFM_MEM_HOST;
  const long long nch = sim_chunk(o->n_draw, Tp, N, r, k, out->F && hst, out->X && hst);
  SsStage s;
  double *gains, *zfS, *fS;
  int* sstat;
  OutSlot<double> oF, oX;
  rc = lay_out(h, [&](Arena& a) {
    s = ss_bufs(a, mem, H, 1, Tp, N, r, p);
    gains = a.get<double>(sim_gains_doubles(Tp, k, r));
    sstat = a.get<int>(1);
    zfS = a.get<double>((size_t)nch * Tp * k);
    fS = a.get<double>((size_t)nch * Tp * r);
    oF = staged(a, out->F, (size_t)Tp * r, nch, hst);
    oX = staged(a, out->X, (size_t)Tp * N, nch, hst);
  });
  if (rc) return rc;
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
    L(k_sim_paths, (nd + SIM_ND - 1) / SIM_ND, 1, SIM_NT, smS, (const double*)gains, src, Tp, r, p, o->seed, id0, nd, (const int*)sstat,
      zfS, fS, oF.at(j0));
    if (out->X)
      L(k_sim_project, ntt, nst * ((nd + SIM_PD - 1) / SIM_PD), 256, smP, s.x, s.pL, s.pR, (const double*)fS, Tp, N, r, o->seed, id0, nd,
        (const int*)sstat, oX.at(j0), 0, 1LL);
    rc = flush(h, j0, nd, mem, oF, oX); if (rc) return rc;
  }
  rc = copy_out(h, out->status, sstat, 1, mem); if (rc) return rc;
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
  SsStage s;
  double *dXn, *dold, *dgv, *dpart, *dbig;
  int *dtg, *dpl, *drowp, *dpst, *dkind;
  unsigned char* dmask;
  OutSlot<double> oOld, oNew, oNews, oW, oC;
  rc = lay_out(h, [&](Arena& a) {
    s = ss_bufs(a, mem, H, B, Tp, N, r, p);
    dXn = dev ? nullptr : a.get<double>(B * onr);
    dtg = a.get<int>(2 * (size_t)nq);
    dmask = a.get<unsigned char>(B * onr);
    dpl = a.get<int>(B * (Wmax + 1));
    drowp = a.get<int>(B * nr);
    dpst = a.get<int>(B);
    dkind = a.get<int>(B * nq);
    dold = a.get<double>(B * nq);
    dgv = a.get<double>(B * nq * nmax);
    dpart = a.get<double>(B * ntile * nq);
    dbig = big_in_smem ? nullptr : a.get<double>(B * bigC);
    oOld = staged(a, out->old_est, (size_t)nq, B, !dev);
    oNew = staged(a, out->new_est, (size_t)nq, B, !dev);
    oNews = staged(a, out->news, onr, B, !dev);
    oW = staged(a, out->weight, onr * nq, B, !dev);
    oC = staged(a, out->contrib, onr * nq, B, !dev);
  });
  if (rc) return rc;
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
  DFM_SET_SMEM(k_news_project, smP);
  const int per = std::max(1, 65535 / nst);          // pairs per launch (grid.y limit)
  for (int b0 = 0; b0 < batch; b0 += per) {
    const int nb = std::min(per, batch - b0);
    L(k_news_project, ntw, nst * nb, 256, smP, (const double*)s.Fs, xn, ldn, row0, s.pL, s.pR, (const unsigned char*)dmask,
      (const int*)drowp, (const double*)dgv, (const int*)dkind, (const int*)dtg, (const int*)dtg + nq, nq, (const int*)dpst, T, Tp, N, r,
      nr, Wmax, b0, oNews.at(0), oW.at(0), oC.at(0), dpart);
  }
  L(k_news_finish, batch, 1, 64, 0, (const double*)dpart, ntile, (const double*)dold, (const int*)dpst, nq, oOld.at(0), oNew.at(0));
  rc = flush(h, 0, B, mem, oOld, oNew, oNews, oW, oC); if (rc) return rc;
  rc = copy_out(h, out->status, dpst, B, mem); if (rc) return rc;
  return finish(h, mem);
}

// ------------------------------------------------------------------------------------ (e)
// ------------------------------------------------------------------------------------ K9: replication generators
int dfm_simulate_panels(dfm_handle* h, unsigned long long seed, long long rep0, int batch, int T, int N, int r, int mem,
                        double* X, double* F_true) {
  if (!h || !X || batch <= 0 || T <= 1 || N <= 0 || r <= 0 || r > 64 || rep0 < 0) return fail(h, DFM_ERR_ARG, "dfm_simulate_panels: bad argument");
  CK(cudaSetDevice(h->device));
  size_t B = batch;
  const bool hst = mem == DFM_MEM_HOST;
  OutSlot<double> oX, oF;
  int rc = lay_out(h, [&](Arena& a) {
    oX = staged(a, X, (size_t)T * N, B, hst);
    oF = scratch(a, F_true, (size_t)T * r, B, hst);
  });
  if (rc) return rc;
  L(k_simulate_panels, batch, 1, 256, 0, seed, rep0, T, N, r, oX.at(0), oF.at(0));
  rc = flush(h, 0, B, mem, oX, oF); if (rc) return rc;
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
  const bool hst = mem == DFM_MEM_HOST;
  double *dF0, *dre, *dbe, *dla, *dac, *dse, *dda;
  OutSlot<double> oX;
  int rc = lay_out(h, [&](Arena& a) {
    dF0 = hst ? a.get<double>((size_t)Tw * r) : nullptr; dre = hst ? a.get<double>((size_t)nres * r) : nullptr;
    dbe = hst ? a.get<double>((size_t)K * r) : nullptr; dla = hst ? a.get<double>((size_t)ns * r) : nullptr;
    dac = hst ? a.get<double>((size_t)ns * Lg) : nullptr; dse = hst ? a.get<double>(ns) : nullptr;
    dda = hst ? a.get<double>((size_t)Tw * ns) : nullptr;
    oX = staged(a, X, (size_t)ns * Tw, B, hst);
  });
  if (rc) return rc;
  BootArgs ba{};
  rc = stage_in(h, F0, dF0, (size_t)Tw * r, mem, &ba.F0); if (rc) return rc;
  rc = stage_in(h, resid, dre, (size_t)nres * r, mem, &ba.resid); if (rc) return rc;
  rc = stage_in(h, beta, dbe, (size_t)K * r, mem, &ba.beta); if (rc) return rc;
  rc = stage_in(h, lam, dla, (size_t)ns * r, mem, &ba.lam); if (rc) return rc;
  rc = stage_in(h, uar_coef, dac, (size_t)ns * Lg, mem, &ba.uar_coef); if (rc) return rc;
  rc = stage_in(h, uar_ser, dse, (size_t)ns, mem, &ba.uar_ser); if (rc) return rc;
  rc = stage_in(h, data, dda, (size_t)Tw * ns, mem, &ba.data); if (rc) return rc;
  ba.X = oX.at(0); ba.Tw = Tw; ba.ns = ns; ba.r = r; ba.p = p; ba.L = Lg; ba.nres = nres; ba.burn = o->burn; ba.seed = o->seed; ba.rep0 = o->rep0;
  DFM_SET_SMEM(k_bootstrap_panels, smem);
  L(k_bootstrap_panels, batch, 1, 256, smem, ba);
  rc = oX.flush(h, 0, B, mem); if (rc) return rc;
  return finish(h, mem);
}

// One call for the whole C4 replication step (SURVEY.md 8b: "one panel + B bootstrap seeds"): resample -> standardise + PCA
// + ALS (estimate_factor!, :328-382) -> sign alignment -> factor VAR (:444-492) -> IRF (:793-825), device resident between
// the stages.  The stages are the public entry points above run on temporaries of this call, which live in the handle's second
// workspace (the stages use and may regrow the first).
int dfm_bootstrap_irf(dfm_handle* h, const dfm_boot_opts* o, const double* F0, const double* resid, const double* beta,
                      const double* lam, const double* uar_coef, const double* uar_ser, const double* data, int nt_min,
                      double tol, int H, double* irf, int* als_iters, int* als_status) {
  if (!h || !o || !F0 || !resid || !beta || !lam || !uar_coef || !uar_ser || !data || !irf || H <= 0)
    return fail(h, DFM_ERR_ARG, "dfm_bootstrap_irf: bad argument");
  const int Tw = o->T, ns = o->ns, r = o->r, p = o->p, Lg = o->n_uarlag, nres = o->n_resid, batch = o->batch, mem = o->mem;
  if (Tw <= p || ns <= 0 || r <= 0 || p <= 0 || Lg <= 0 || nres <= 0 || batch <= 0) return fail(h, DFM_ERR_ARG, "dfm_bootstrap_irf: bad shape");
  CK(cudaSetDevice(h->device));
  const size_t B = batch; const int k = r * p, K = 1 + k;
  const bool hst = mem == DFM_MEM_HOST;
  const size_t nin[7] = {(size_t)Tw * r, (size_t)nres * r, (size_t)K * r, (size_t)ns * r, (size_t)ns * Lg, (size_t)ns, (size_t)Tw * ns};
  const double* hin[7] = {F0, resid, beta, lam, uar_coef, uar_ser, data};
  double* dIn[7];
  double *dX, *dF, *dM, *dQ, *dG;
  OutSlot<double> oI;
  int rc = lay_out(h, [&](Arena& a) {
    for (int i = 0; i < 7; ++i) dIn[i] = hst ? a.get<double>(nin[i]) : nullptr;
    dX = a.get<double>(B * ns * Tw); dF = a.get<double>(B * Tw * r);
    dM = a.get<double>(B * k * k); dQ = a.get<double>(B * r * k); dG = a.get<double>(B * k * r);
    oI = staged(a, irf, (size_t)r * H * r, B, hst);
  }, true);
  if (rc) return rc;
  // the stages; a failure after work is queued drains the stream before it returns
  const int ret = [&]() -> int {
    const double* din[7];
    for (int i = 0; i < 7; ++i)            // (any mem but DFM_MEM_HOST reads the inputs in place)
      if (stage_in(h, hin[i], dIn[i], nin[i], hst ? DFM_MEM_HOST : DFM_MEM_DEVICE, &din[i]))
        return fail(h, DFM_ERR_CUDA, "dfm_bootstrap_irf: upload failed");
    dfm_boot_opts ob = *o; ob.mem = DFM_MEM_DEVICE;
    rc = dfm_bootstrap_panels(h, &ob, din[0], din[1], din[2], din[3], din[4], din[5], din[6], dX);
    if (rc) return rc;
    dfm_factor_opts fo{}; fo.T = Tw; fo.N = ns; fo.r = r; fo.nt_min = nt_min; fo.tol = tol; fo.max_iter = 100000000; fo.compute_r2 = 0;
    fo.n_constr = 0; fo.batch = batch; fo.mem = DFM_MEM_DEVICE;
    std::vector<dfm_factor_stats> fs(B);
    rc = dfm_estimate_factor(h, dX, &fo, nullptr, dF, nullptr, nullptr, nullptr, nullptr, fs.data());
    if (rc) return rc;
    for (size_t b = 0; b < B; ++b) { if (als_iters) als_iters[b] = fs[b].iters; if (als_status) als_status[b] = fs[b].status; }
    L(k_sign_align, batch, 1, 128, 48 * 8, dF, din[0], Tw, r);
    rc = dfm_estimate_var(h, dF, Tw, r, p, 1, batch, DFM_MEM_DEVICE, nullptr, nullptr, nullptr, dM, dQ, dG);
    if (rc != DFM_OK && rc != DFM_ERR_NOT_PD && rc != DFM_ERR_TOO_FEW_OBS) return rc;       // (all panels failed: records stay NaN)
    std::vector<int> ids(r); for (int j = 0; j < r; ++j) ids[j] = j;
    rc = dfm_irf(h, dM, dQ, dG, k, r, H, r, ids.data(), batch, DFM_MEM_DEVICE, oI.at(0));
    if (rc) return rc;
    if (oI.flush(h, 0, B, mem)) return fail(h, DFM_ERR_CUDA, "dfm_bootstrap_irf: download failed");
    return DFM_OK;
  }();
  cudaError_t e = cudaStreamSynchronize(h->stream);
  if (ret) return ret;
  CK(e);
  return DFM_OK;
}

// ------------------------------------------------------------------------------------ parametric bootstrap (state-space model)
// k_ss_simulate, then k_ss_sim_project in launches of at most 65535 / ceil(N / SS_NS) tiles of SIM_PD replicates (grid.y).
// g: the factors of k_ss_sim_chol; fS: nb * T * r scratch; Xout: nb panels.
static void ssb_simulate(dfm_handle* h, const double* xt, const double* Lam, const double* Rv, const double* g, int T, int N, int r, int p,
                         unsigned long long seed, long long rep0, int nb, double* fS, double* Xout) {
  const size_t smS = ssb_sim_smem_doubles(r, p) * 8, smP = ssb_project_smem_doubles(r) * 8;
  DFM_SET_SMEM(k_ss_simulate, smS);
  DFM_SET_SMEM(k_ss_sim_project, smP);
  L(k_ss_simulate, (nb + SSB_ND - 1) / SSB_ND, 1, SSB_NT, smS, g, T, r, p, seed, rep0, nb, fS);
  const int nst = (N + SS_NS - 1) / SS_NS, ntt = (T + SS_TP - 1) / SS_TP;
  const int per = std::max(1, 65535 / nst) * SIM_PD;
  for (int j0 = 0; j0 < nb; j0 += per) {
    const int n = std::min(per, nb - j0);
    L(k_ss_sim_project, ntt, nst * ((n + SIM_PD - 1) / SIM_PD), 256, smP, xt, Lam, Rv, (const double*)(fS + (size_t)j0 * T * r), T, N, r,
      seed, rep0 + j0, n, Xout + (size_t)j0 * T * N);
  }
}

int dfm_ss_simulate_panels(dfm_handle* h, const double* X, int T, int N, int r, int p, const dfm_em_init* params, unsigned long long seed,
                           long long rep0, int batch, int mem, double* Xout) {
  if (!h || !X || !params || !Xout || !params->Lam || !params->R || !params->A || !params->Q || !params->P0)
    return fail(h, DFM_ERR_ARG, "dfm_ss_simulate_panels: null argument (P0 is required)");
  if (T <= 1 || N <= 0 || r <= 0 || p <= 0 || batch <= 0 || rep0 < 0 || (mem != DFM_MEM_HOST && mem != DFM_MEM_DEVICE))
    return fail(h, DFM_ERR_ARG, "dfm_ss_simulate_panels: bad shape/options");
  if (r * p > 48) return fail(h, DFM_ERR_UNSUPPORTED, "dfm_ss_simulate_panels: state dimension r*p > 48");
  CK(cudaSetDevice(h->device));
  const size_t B = batch, TN = (size_t)T * N; const int k = r * p;
  const bool hst = mem == DFM_MEM_HOST;
  double *dX, *dL, *dR, *dA, *dQ, *dP, *g, *fS;
  OutSlot<double> oX;
  int rc = lay_out(h, [&](Arena& a) {
    dX = hst ? a.get<double>(TN) : nullptr;
    dL = hst ? a.get<double>((size_t)N * r) : nullptr; dR = hst ? a.get<double>(N) : nullptr;
    dA = hst ? a.get<double>((size_t)r * k) : nullptr; dQ = hst ? a.get<double>((size_t)r * r) : nullptr;
    dP = hst ? a.get<double>((size_t)k * k) : nullptr;
    g = a.get<double>(ssb_chol_doubles(r, p));
    fS = a.get<double>(B * T * r);
    oX = staged(a, Xout, TN, B, hst);
  });
  if (rc) return rc;
  const double *x, *l, *rv, *am, *q, *p0;
  rc = stage_in(h, X, dX, TN, mem, &x); if (rc) return rc;
  rc = stage_in(h, params->Lam, dL, (size_t)N * r, mem, &l); if (rc) return rc;
  rc = stage_in(h, params->R, dR, (size_t)N, mem, &rv); if (rc) return rc;
  rc = stage_in(h, params->A, dA, (size_t)r * k, mem, &am); if (rc) return rc;
  rc = stage_in(h, params->Q, dQ, (size_t)r * r, mem, &q); if (rc) return rc;
  rc = stage_in(h, params->P0, dP, (size_t)k * k, mem, &p0); if (rc) return rc;
  L(k_ss_sim_chol, 1, 1, 128, ssb_chol_smem_doubles(r, p) * 8, am, q, p0, r, p, g);
  ssb_simulate(h, x, l, rv, g, T, N, r, p, seed, rep0, batch, fS, oX.at(0));
  rc = oX.flush(h, 0, B, mem); if (rc) return rc;
  return finish(h, mem);
}

// Replicates per sub-batch of dfm_ss_bootstrap: a function of the model's shape and the device only, never of n_rep, rep0 or
// the outputs asked for.  dfm_em_kalman and dfm_kalman_smooth choose their launch plan (thread-block cluster, threads, staging
// tile, multi-CTA contraction split) from their batch, and plans sum in different orders; every sub-batch therefore has
// exactly this many replicates (the last one is filled with the replication ids that follow), so that a replicate's results
// are the same bits whatever n_rep, the shard split or the number of calls.  At most two waves of the fused kernels' grid
// (2 CTAs per SM), and the device memory an estimate of a sub-batch needs (panel, factors, parameter copies and the EM's
// general-path workspace per replicate) within kSimChunkBytes.
static int ssb_batch(const dfm_handle* h, int T, int N, int r, int p) {
  const size_t k = (size_t)r * p, kk = k * k, rk = r * k, np = (size_t)r * (r + 1) / 2;
  const size_t par = (size_t)N * r + N + rk + (size_t)r * r;
  const size_t per = 8 * ((size_t)T * N + (size_t)T * r + 8 * par + 3 * kk + (size_t)T * (2 * kk + 2 * k + 2 * np + 4 * r + 4) + 64 * k +
                          16 * (kk + rk));
  const long long cap = std::max<long long>(1, (long long)(kSimChunkBytes / per));
  return (int)std::min<long long>(cap, std::min(2 * h->nsm, kMaxGridBatch));
}

// The whole parametric bootstrap, per sub-batch of ssb_batch() replicates: k_ss_simulate (+ k_ss_sim_project) -> dfm_em_kalman
// from the fitted parameters -> k_ss_align -> dfm_irf -> (forecasts) copies of the panel, dfm_kalman_smooth at the aligned
// parameters and k_ss_fc_rows.  The stages are the public entry points run on temporaries of this call, which live in the
// handle's second workspace (the stages use and may regrow the first); the device memory does not grow with n_rep.
int dfm_ss_bootstrap(dfm_handle* h, const double* X, const dfm_ssb_opts* o, const dfm_em_init* params, const dfm_ssb_out* out) {
  if (!h || !X || !o || !params || !out || !params->Lam || !params->R || !params->A || !params->Q || !params->P0)
    return fail(h, DFM_ERR_ARG, "dfm_ss_bootstrap: null argument (P0 is required)");
  const int T = o->T, N = o->N, r = o->r, p = o->p, Hi = o->H_irf, Hf = o->H_fc, fr = o->fc_rows, mi = o->max_iter, mem = o->mem;
  const long long n_rep = o->n_rep;
  if (T <= 1 || N <= 0 || r <= 0 || p <= 0 || Hi <= 0 || Hf < 0 || fr < 0 || (long long)fr > (long long)T + Hf || mi <= 0 ||
      !(o->tol >= 0) || n_rep < 1 || o->rep0 < 0 || (mem != DFM_MEM_HOST && mem != DFM_MEM_DEVICE))
    return fail(h, DFM_ERR_ARG, "dfm_ss_bootstrap: bad shape/options");
  const int k = r * p;
  if (k > 48) return fail(h, DFM_ERR_UNSUPPORTED, "dfm_ss_bootstrap: state dimension r*p > 48");
  const bool fc = fr > 0 && (out->xhat || out->xvar);
  const int Tp = T + Hf;
  const int nc = ssb_batch(h, T, N, r, p);
  if (em_fs_smem_doubles(r, p, fs_stage_periods(h->nsm, nc, r, p)) * 8 > kMaxSmem)
    return fail(h, DFM_ERR_UNSUPPORTED, "dfm_ss_bootstrap: state dimension r*p too large for the general path");
  CK(cudaSetDevice(h->device));
  const size_t B = nc, TN = (size_t)T * N, kk = (size_t)k * k, rr = (size_t)r * r, rk = (size_t)r * k, Nr = (size_t)N * r;
  const size_t nirf = (size_t)r * Hi * r;
  const bool hst = mem == DFM_MEM_HOST;
  // temporaries of this call, in the second workspace (the stages' own scratch lives in the first, which they may regrow).  Every
  // sub-batch computes nc replicates and returns nkeep of them, so the records always go through their buffers.
  double *dXs, *dLh, *dRh, *dAh, *dQh, *dPh, *g, *dX, *fS, *iL, *iR, *iA, *iQ, *iP, *eL, *eR, *eA, *eQ, *ell, *pL, *pR, *pA, *pQ, *dM,
      *dQs, *dG, *xh, *xv;
  int *eit, *est;
  OutSlot<double> oL, oR, oA, oQ, oI, oFh, oFv, oLl;
  OutSlot<int> oIt, oSt;
  int rc = lay_out(h, [&](Arena& a) {
    dXs = hst ? a.get<double>(TN) : nullptr; dLh = hst ? a.get<double>(Nr) : nullptr; dRh = hst ? a.get<double>(N) : nullptr;
    dAh = hst ? a.get<double>(rk) : nullptr; dQh = hst ? a.get<double>(rr) : nullptr; dPh = hst ? a.get<double>(kk) : nullptr;
    g = a.get<double>(ssb_chol_doubles(r, p));
    dX = a.get<double>(B * TN); fS = a.get<double>(B * T * r);
    iL = a.get<double>(B * Nr); iR = a.get<double>(B * N); iA = a.get<double>(B * rk); iQ = a.get<double>(B * rr); iP = a.get<double>(B * kk);
    eL = a.get<double>(B * Nr); eR = a.get<double>(B * N); eA = a.get<double>(B * rk); eQ = a.get<double>(B * rr); ell = a.get<double>(B * mi);
    eit = a.get<int>(B); est = a.get<int>(B);
    oL = {out->Lam, a.get<double>(B * Nr), Nr}; oR = {out->R, a.get<double>(B * N), (size_t)N};
    oA = {out->A, a.get<double>(B * rk), rk}; oQ = {out->Q, a.get<double>(B * rr), rr};
    pL = fc ? a.get<double>(B * Nr) : nullptr; pR = fc ? a.get<double>(B * N) : nullptr;
    pA = fc ? a.get<double>(B * rk) : nullptr; pQ = fc ? a.get<double>(B * rr) : nullptr;
    dM = a.get<double>(B * kk); dQs = a.get<double>(B * rk); dG = a.get<double>(B * rk);
    oLl = {out->loglik, a.get<double>(B), 1}; oSt = {out->status, a.get<int>(B), 1};
    oI = {out->irf, a.get<double>(B * nirf), nirf};
    xh = fc ? a.get<double>(B * Tp * N) : nullptr; xv = fc ? a.get<double>(B * Tp * N) : nullptr;
    oFh = {out->xhat, fc ? a.get<double>(B * fr * N) : nullptr, (size_t)fr * N};
    oFv = {out->xvar, fc ? a.get<double>(B * fr * N) : nullptr, (size_t)fr * N};
    oIt = {out->iters, eit, 1};
  }, true);
  if (rc) return rc;
  // the sub-batches; a failure after work is queued drains the stream before it returns
  const int ret = [&]() -> int {
    const double *xs, *Lh, *Rh, *Ah, *Qh, *Ph;
    if (stage_in(h, X, dXs, TN, mem, &xs) || stage_in(h, params->Lam, dLh, Nr, mem, &Lh) ||
        stage_in(h, params->R, dRh, (size_t)N, mem, &Rh) || stage_in(h, params->A, dAh, rk, mem, &Ah) ||
        stage_in(h, params->Q, dQh, rr, mem, &Qh) || stage_in(h, params->P0, dPh, kk, mem, &Ph))
      return fail(h, DFM_ERR_CUDA, "dfm_ss_bootstrap: copy failed");
    L(k_ss_sim_chol, 1, 1, 128, ssb_chol_smem_doubles(r, p) * 8, Ah, Qh, Ph, r, p, g);
    std::vector<int> ids(r);
    for (int j = 0; j < r; ++j) ids[j] = j;
    const size_t smA = ssb_align_smem_doubles(r, p) * 8;
    DFM_SET_SMEM(k_ss_align, smA);
    auto bcast = [&](const double* src, size_t n, double* dst, int nb) {
      L(k_ss_bcast, (int)std::min<size_t>((n + 255) / 256, 1024), nb, 256, 0, src, (long long)n, dst);
    };
    for (long long j0 = 0; j0 < n_rep; j0 += nc) {
      const int nb = nc;                                              // replicates computed (a full sub-batch, see ssb_batch)
      const int nkeep = (int)std::min<long long>(nc, n_rep - j0);     // ... and returned
      // 1. panels
      ssb_simulate(h, xs, Lh, Rh, g, T, N, r, p, o->seed, o->rep0 + j0, nb, fS, dX);
      // 2. EM from the fitted parameters (P0 held fixed)
      bcast(Lh, Nr, iL, nb); bcast(Rh, N, iR, nb); bcast(Ah, rk, iA, nb); bcast(Qh, rr, iQ, nb); bcast(Ph, kk, iP, nb);
      dfm_em_opts eo{}; eo.T = T; eo.N = N; eo.r = r; eo.p = p; eo.max_iter = mi; eo.tol = o->tol; eo.batch = nb; eo.mem = DFM_MEM_DEVICE; eo.path = 0;
      dfm_em_init ei{iL, iR, iA, iQ, iP};
      dfm_em_out eout{}; eout.Lam = eL; eout.R = eR; eout.A = eA; eout.Q = eQ; eout.loglik = ell; eout.iters = eit; eout.status = est;
      rc = dfm_em_kalman(h, dX, &eo, &ei, &eout);
      if (rc) return rc;
      // 3. alignment
      SsbAlignArgs aa{};
      aa.Lh = Lh; aa.Rh = Rh; aa.Ah = Ah; aa.Qh = Qh;
      aa.Ls = eL; aa.Rs = eR; aa.As = eA; aa.Qs = eQ; aa.ll = ell; aa.it = eit; aa.em_status = est;
      aa.Lo = oL.buf; aa.Ro = oR.buf; aa.Ao = oA.buf; aa.Qo = oQ.buf;
      if (fc) { aa.Le = pL; aa.Re = pR; aa.Ae = pA; aa.Qe = pQ; }
      aa.M = dM; aa.Qsel = dQs; aa.G = dG; aa.llf = oLl.buf; aa.status = oSt.buf;
      aa.N = N; aa.r = r; aa.p = p; aa.max_iter = mi;
      L(k_ss_align, nb, 1, SSB_NT, smA, aa);
      // 4. impulse responses of all r shocks
      rc = dfm_irf(h, dM, dQs, dG, k, r, Hi, r, ids.data(), nb, DFM_MEM_DEVICE, oI.buf);
      if (rc) return rc;
      // 5. forecasts: the original panel at every replicate's aligned parameters
      if (fc) {
        bcast(xs, TN, dX, nb);
        dfm_ss_opts so{}; so.T = T; so.N = N; so.r = r; so.p = p; so.H = Hf; so.batch = nb; so.mem = DFM_MEM_DEVICE;
        dfm_em_init sp{pL, pR, pA, pQ, iP};
        dfm_ss_out sout{}; sout.xhat = xh; sout.xvar = xv;
        rc = dfm_kalman_smooth(h, dX, &so, &sp, &sout);
        if (rc) return rc;
        const long long n = (long long)nb * N * fr;
        L(k_ss_fc_rows, (int)std::min<long long>((n + 255) / 256, 4096), 1, 256, 0, (const double*)xh, (const double*)xv, Tp, N, fr, nb,
          (const int*)oSt.buf, out->xhat ? oFh.buf : (double*)nullptr, out->xvar ? oFv.buf : (double*)nullptr);
      }
      // 6. records
      rc = flush(h, j0, nkeep, mem, oL, oR, oA, oQ, oI);
      if (!rc && fc) rc = flush(h, j0, nkeep, mem, oFh, oFv);
      if (!rc) rc = flush(h, j0, nkeep, mem, oLl, oIt, oSt);
      if (rc || cudaGetLastError() != cudaSuccess) return fail(h, DFM_ERR_CUDA, "dfm_ss_bootstrap: copy failed");
    }
    return DFM_OK;
  }();
  cudaError_t e = cudaStreamSynchronize(h->stream);
  if (ret) return ret;
  CK(e);
  return DFM_OK;
}

// ------------------------------------------------------------------------------------ Gibbs sampler
// Per sub-batch of ssb_batch() chains (the bootstrap's rule: a size fixed by the model's shape and the device, so that chain c
// has the same bits whatever n_chain or chain0), the sweeps run device-resident with no host synchronisation between them
// (records going to pageable host memory are staged per kept sweep):
//   ss_estep (one padded panel copy per chain, k_ss_bcast once per call) -> k_sim_gains (grid.y = chain) -> k_gibbs_paths ->
//   [kept: k_sim_project + k_ss_fc_rows] -> k_gibbs_stats -> k_gibbs_draw -> [kept: records, k_ss_align + k_irf].
// dfm_gibbs and dfm_gibbs_constrained.  con == nullptr or con->n_constr == 0: the unrestricted sampler (same launches, same
// bits).  Otherwise the rows are checked as dfm_em_kalman_constrained's, uploaded once as a per-series CSR, and the parameter
// step is k_gibbs_draw_constr.
static int gibbs_impl(dfm_handle* h, const double* X, const dfm_gibbs_opts* o, const dfm_em_init* init, const dfm_em_init* ref,
                      const dfm_lam_constr* con, const dfm_gibbs_out* out) {
  if (!h || !X || !o || !init || !out || !init->Lam || !init->R || !init->A || !init->Q || !init->P0)
    return fail(h, DFM_ERR_ARG, "dfm_gibbs: null argument (P0 is required)");
  const int T = o->T, N = o->N, r = o->r, p = o->p, Hi = o->H_irf, Hf = o->H_fc, fr = o->fc_rows, mem = o->mem;
  const long long nch = o->n_chain;
  const dfm_gibbs_prior& pr = o->prior;
  if (T <= 1 || N <= 0 || r <= 0 || p <= 0 || Hi < 0 || Hf < 0 || fr < 0 || (long long)fr > (long long)T + Hf || nch < 1 ||
      o->chain0 < 0 || o->chain0 + nch > (1LL << 16) || o->sweep0 < 0 || o->n_burn < 0 || o->n_keep < 1 || o->thin < 1 ||
      (mem != DFM_MEM_HOST && mem != DFM_MEM_DEVICE))
    return fail(h, DFM_ERR_ARG, "dfm_gibbs: bad shape/options");
  const long long n_sweep = (long long)o->n_burn + (long long)o->n_keep * o->thin;
  if (o->sweep0 + n_sweep > (1LL << 24)) return fail(h, DFM_ERR_ARG, "dfm_gibbs: sweep indices must stay below 2^24");
  if (!(pr.kap_lam > 0) || !(pr.a_R >= 1) || !(pr.b_R > 0) || !(pr.kap_A > 0) || !(pr.s_Q > 0) || !(pr.nu_Q + T - r >= 2) ||
      !std::isfinite(pr.kap_lam + pr.a_R + pr.b_R + pr.kap_A + pr.nu_Q + pr.s_Q))
    return fail(h, DFM_ERR_ARG, "dfm_gibbs: bad prior (kappas, b_R, s_Q > 0, a_R >= 1, nu_Q + T - r >= 2)");
  if (Hi > 0 && out->irf && (!ref || !ref->Lam || !ref->R || !ref->A || !ref->Q))
    return fail(h, DFM_ERR_ARG, "dfm_gibbs: ref is required for impulse responses");
  ConstrCsr cc;
  { int rc = constr_csr(h, "dfm_gibbs_constrained", con, N, r, &cc); if (rc) return rc; }
  if (cc.nc && out->irf)
    return fail(h, DFM_ERR_ARG, "dfm_gibbs_constrained: no impulse responses with restrictions (the rotation onto ref would undo them)");
  const int k = r * p, Tp = T + Hf;
  if (k > 48) return fail(h, DFM_ERR_UNSUPPORTED, "dfm_gibbs: state dimension r*p > 48");
  const int C = ssb_batch(h, T, N, r, p);
  int rc = ss_check(h, "dfm_gibbs", Tp, N, r, p, 0, C, DFM_MEM_DEVICE);
  if (rc) return rc;
  const size_t smG = sim_gains_smem_doubles(r, p) * 8, smPa = gibbs_paths_smem_doubles(r, p) * 8, smSt = gibbs_stats_smem_doubles() * 8,
               smD = gibbs_draw_smem_doubles(r, p) * 8, smP = sim_project_smem_doubles(r) * 8, smA = ssb_align_smem_doubles(r, p) * 8,
               smI = irf_smem_doubles(k) * 8;
  if (smD > kMaxSmem) return fail(h, DFM_ERR_UNSUPPORTED, "dfm_gibbs: state too large for the parameter-draw kernel");
  const size_t smDc = smD + gibbs_constr_smem_doubles(r) * 8;          // k_gibbs_draw_constr
  if (cc.nc && smDc > kMaxSmem) return fail(h, DFM_ERR_UNSUPPORTED, "dfm_gibbs_constrained: state too large for the parameter-draw kernel");
  const int nst = (N + SS_NS - 1) / SS_NS;
  if ((long long)nst * ((C + SIM_PD - 1) / SIM_PD) > kMaxGridBatch) return fail(h, DFM_ERR_UNSUPPORTED, "dfm_gibbs: N too large");
  CK(cudaSetDevice(h->device));
  const size_t B = C, Nr = (size_t)N * r, rk = (size_t)r * k, rr = (size_t)r * r, kk = (size_t)k * k, nirf = (size_t)r * Hi * r;
  const bool wantX = out->X && fr > 0, wantI = out->irf && Hi > 0;
  const bool hst = mem == DFM_MEM_HOST;
  const cudaMemcpyKind kin = hst ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToDevice, kout = hst ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice;
  const long long nk = o->n_keep;
  SsStage s;
  double *Xpad, *dL, *dR, *dA, *dQ, *dP, *gains, *zfS, *fS, *z0, *sv, *wk, *qv, *Fk, *Xproj, *Xrow, *sL, *sR, *sA, *sQ, *sll, *rL, *rR,
      *rA, *rQ, *aL, *aR, *aA, *aQ, *aM, *aS, *aG, *allf, *adum, *dI;
  int *cst, *nobs, *mcnt, *midx, *sst, *ast, *ids;
  EmConstr cs;
  rc = lay_out(h, [&](Arena& a) {
    s = ss_bufs(a, DFM_MEM_DEVICE, 0, B, Tp, N, r, p);
    Xpad = a.get<double>(B * Tp * N);
    dL = a.get<double>(B * Nr); dR = a.get<double>(B * N); dA = a.get<double>(B * rk); dQ = a.get<double>(B * rr);
    dP = a.get<double>(B * kk);
    gains = a.get<double>(B * sim_gains_doubles(Tp, k, r));
    cst = a.get<int>(B);
    zfS = a.get<double>(B * Tp * k); fS = a.get<double>(B * Tp * r); z0 = a.get<double>(B * k); sv = a.get<double>(B * Nr);
    wk = a.get<double>(B * gibbs_draw_wk_doubles(N, r));
    nobs = a.get<int>(N); mcnt = a.get<int>(N); midx = a.get<int>((size_t)N * T);
    qv = a.get<double>(N);
    Fk = out->F ? a.get<double>(B * Tp * r) : nullptr;
    Xproj = wantX ? a.get<double>(B * Tp * N) : nullptr;
    Xrow = wantX ? a.get<double>(B * fr * N) : nullptr;
    sL = a.get<double>(B * Nr); sR = a.get<double>(B * N); sA = a.get<double>(B * rk); sQ = a.get<double>(B * rr);
    sll = a.get<double>(B);
    sst = a.get<int>(B);
    rL = wantI ? a.get<double>(Nr) : nullptr; rR = wantI ? a.get<double>(N) : nullptr; rA = wantI ? a.get<double>(rk) : nullptr;
    rQ = wantI ? a.get<double>(rr) : nullptr;
    aL = wantI ? a.get<double>(B * Nr) : nullptr; aR = wantI ? a.get<double>(B * N) : nullptr;
    aA = wantI ? a.get<double>(B * rk) : nullptr; aQ = wantI ? a.get<double>(B * rr) : nullptr;
    aM = wantI ? a.get<double>(B * kk) : nullptr; aS = wantI ? a.get<double>(B * rk) : nullptr;
    aG = wantI ? a.get<double>(B * rk) : nullptr; allf = wantI ? a.get<double>(B) : nullptr;
    adum = wantI ? a.get<double>(B + 4) : nullptr; dI = wantI ? a.get<double>(B * nirf) : nullptr;
    ast = wantI ? a.get<int>(B) : nullptr;
    ids = wantI ? a.get<int>(r) : nullptr;
    cs = constr_bufs(a, cc, N, r);
  });
  if (rc) return rc;
  rc = constr_upload(h, cc, cs);
  if (rc) return rc;
  // ---- once per call: the padded panel, its copies, the per-series counts; the reference model and shock ids
  if (hst) {
    CK(cudaMemcpy2DAsync(Xpad, (size_t)Tp * 8, X, (size_t)T * 8, (size_t)T * 8, N, cudaMemcpyHostToDevice, h->stream));
    if (Hf > 0) L(k_ss_pad, (int)std::min<long long>(((long long)N * Hf + 255) / 256, 4096), 1, 256, 0, (const double*)nullptr, T, Tp, (long long)N, Xpad);
  } else {
    L(k_ss_pad, (int)std::min<long long>(((long long)N * Tp + 255) / 256, 4096), 1, 256, 0, X, T, Tp, (long long)N, Xpad);
  }
  auto bcast = [&](const double* src, size_t n, double* dst, int nb) {
    if (nb > 0) L(k_ss_bcast, (int)std::min<size_t>((n + 255) / 256, 1024), nb, 256, 0, src, (long long)n, dst);
  };
  bcast(Xpad, (size_t)Tp * N, Xpad + (size_t)Tp * N, C - 1);
  L(k_gibbs_scan, (N + 127) / 128, 1, 128, 0, (const double*)Xpad, T, Tp, N, nobs, qv, mcnt, midx);
  if (wantI) {
    CK(cudaMemcpyAsync(rL, ref->Lam, Nr * 8, kin, h->stream)); CK(cudaMemcpyAsync(rR, ref->R, (size_t)N * 8, kin, h->stream));
    CK(cudaMemcpyAsync(rA, ref->A, rk * 8, kin, h->stream)); CK(cudaMemcpyAsync(rQ, ref->Q, rr * 8, kin, h->stream));
    std::vector<int> hid(r);
    for (int j = 0; j < r; ++j) hid[j] = j;
    CK(cudaMemcpyAsync(ids, hid.data(), r * sizeof(int), cudaMemcpyHostToDevice, h->stream));
    CK(cudaStreamSynchronize(h->stream));                  // (hid is a local)
    DFM_SET_SMEM(k_ss_align, smA);
    DFM_SET_SMEM(k_irf, smI);
  }
  DFM_SET_SMEM(k_sim_gains, smG);
  DFM_SET_SMEM(k_gibbs_paths, smPa);
  DFM_SET_SMEM(k_gibbs_stats, smSt);
  if (cc.nc) DFM_SET_SMEM(k_gibbs_draw_constr, smDc);
  else DFM_SET_SMEM(k_gibbs_draw, smD);
  DFM_SET_SMEM(k_sim_project, smP);
  const int* src = s.g.nt + (size_t)C * Tp;
  const long long idstride = 1LL << 24;
  GibbsDrawArgs da{};
  da.X = Xpad; da.fS = fS; da.z0 = z0; da.sv = sv; da.q = qv; da.nobs = nobs; da.mcnt = mcnt; da.midx = midx;
  da.Lam = dL; da.R = dR; da.A = dA; da.Q = dQ; da.wk = wk; da.cst = cst;
  da.pr = GbPrior{pr.kap_lam, pr.a_R, pr.b_R, pr.kap_A, pr.nu_Q, pr.s_Q};
  da.T = T; da.Tp = Tp; da.N = N; da.r = r; da.p = p; da.C = C; da.seed = o->seed; da.idstride = idstride;
  for (long long j0 = 0; j0 < nch; j0 += C) {
    const int nkeep = (int)std::min<long long>(C, nch - j0);       // chains returned (a full sub-batch is computed)
    // ---- initial parameters: the sub-batch's chains, then copies of the last chain's for the fill-up
    const double* isrc[5] = {init->Lam, init->R, init->A, init->Q, init->P0};
    double* idst[5] = {dL, dR, dA, dQ, dP};
    const size_t isz[5] = {Nr, (size_t)N, rk, rr, kk};
    for (int q = 0; q < 5; ++q) {
      CK(cudaMemcpyAsync(idst[q], isrc[q] + (size_t)j0 * isz[q], (size_t)nkeep * isz[q] * 8, kin, h->stream));
      bcast(idst[q] + (size_t)(nkeep - 1) * isz[q], isz[q], idst[q] + (size_t)nkeep * isz[q], C - nkeep);
    }
    CK(cudaMemsetAsync(cst, 0, B * sizeof(int), h->stream));
    // ---- records: rows [j0, j0 + nkeep) of an output with `per` elements per chain, at element offset `off` of each row
    cudaError_t ce = cudaSuccess;
    auto put = [&](void* dst, const void* srcd, size_t n, size_t esz, size_t per, size_t off) {
      if (dst && ce == cudaSuccess)
        ce = cudaMemcpy2DAsync((char*)dst + ((size_t)j0 * per + off) * esz, per * esz, srcd, n * esz, n * esz, nkeep, kout, h->stream);
    };
    const long long cid0 = o->chain0 + j0;
    for (long long sw = 0; sw < n_sweep; ++sw) {
      const bool kept = sw >= o->n_burn && (sw - o->n_burn + 1) % o->thin == 0;
      const long long jk = kept ? (sw - o->n_burn + 1) / o->thin - 1 : -1;
      const long long id0 = (cid0 << 24) + o->sweep0 + sw;
      dfm_em_init ep{dL, dR, dA, dQ, dP};
      rc = ss_estep(h, s, Xpad, &ep, Tp, N, r, p, 0, C, DFM_MEM_DEVICE);
      if (rc) return rc;
      L(k_sim_gains, Tp + 1, C, 256, smG, s.pA, s.pQ, (const double*)s.P0, (const double*)s.g.C, (const double*)s.g.Ct,
        (const double*)s.g.Bt, (const double*)s.g.Pp, (const double*)s.g.Pf, src, (const int*)s.g.nt, (const EmState*)s.st, Tp, r, p,
        gains, cst);
      L(k_gibbs_paths, (C + GB_PW - 1) / GB_PW, 1, 32 * GB_PW, smPa, (const double*)gains, Tp, r, p, C, o->seed, id0, idstride,
        (const int*)cst, zfS, fS, z0, kept ? Fk : (double*)nullptr);
      if (out->loglik) {
        L(k_gibbs_rec, 1, C, 32, 0, (const double*)s.ll, 1LL, 1LL, (const int*)cst, sll, 1LL);
        put(out->loglik, sll, 1, 8, (size_t)n_sweep, (size_t)sw);
      }
      if (kept && wantX) {
        L(k_sim_project, (Tp + SS_TP - 1) / SS_TP, nst * ((C + SIM_PD - 1) / SIM_PD), 256, smP, (const double*)Xpad, (const double*)dL,
          (const double*)dR, (const double*)fS, Tp, N, r, o->seed, id0, C, (const int*)cst, Xproj, 1, idstride);
        const long long n = (long long)C * N * fr;
        L(k_ss_fc_rows, (int)std::min<long long>((n + 255) / 256, 4096), 1, 256, 0, (const double*)Xproj, (const double*)nullptr, Tp, N,
          fr, C, (const int*)cst, Xrow, (double*)nullptr);
      }
      L(k_gibbs_stats, (N + GB_NS - 1) / GB_NS, (C * r + GB_NC - 1) / GB_NC, 128, smSt, (const double*)Xpad, (const double*)fS, T, Tp, N,
        r, C, sv);
      da.id0 = id0;
      if (cc.nc) L(k_gibbs_draw_constr, C, 1, GB_NT, smDc, da, cs);
      else L(k_gibbs_draw, C, 1, GB_NT, smD, da);
      if (kept) {
        const double* psrc[4] = {dL, dR, dA, dQ};
        double* pst[4] = {sL, sR, sA, sQ};
        double* pdst[4] = {out->Lam, out->R, out->A, out->Q};
        for (int q = 0; q < 4; ++q) {
          if (!pdst[q]) continue;
          L(k_gibbs_rec, (int)std::min<size_t>((isz[q] + 255) / 256, 64), C, 256, 0, psrc[q], (long long)isz[q], (long long)isz[q],
            (const int*)cst, pst[q], (long long)isz[q]);
          put(pdst[q], pst[q], isz[q], 8, (size_t)nk * isz[q], (size_t)jk * isz[q]);
        }
        if (out->F) put(out->F, Fk, (size_t)Tp * r, 8, (size_t)nk * Tp * r, (size_t)jk * Tp * r);
        if (wantX) put(out->X, Xrow, (size_t)fr * N, 8, (size_t)nk * fr * N, (size_t)jk * fr * N);
        if (wantI) {
          SsbAlignArgs aa{};
          aa.Lh = rL; aa.Rh = rR; aa.Ah = rA; aa.Qh = rQ;
          aa.Ls = dL; aa.Rs = dR; aa.As = dA; aa.Qs = dQ;
          aa.ll = adum; aa.it = cst; aa.em_status = cst;        // (it = status in {0, 3}: llf reads adum[b + 2] at most)
          aa.Lo = aL; aa.Ro = aR; aa.Ao = aA; aa.Qo = aQ;
          aa.M = aM; aa.Qsel = aS; aa.G = aG; aa.llf = allf; aa.status = ast;
          aa.N = N; aa.r = r; aa.p = p; aa.max_iter = 1;
          L(k_ss_align, C, 1, SSB_NT, smA, aa);
          L(k_irf, r, C, 64, smI, (const double*)aM, (const double*)aS, (const double*)aG, k, r, Hi, r, (const int*)ids, dI);
          put(out->irf, dI, nirf, 8, (size_t)nk * nirf, (size_t)jk * nirf);
        }
      }
      if (ce != cudaSuccess) { cudaStreamSynchronize(h->stream); return fail(h, DFM_ERR_CUDA, "dfm_gibbs: copy failed"); }
    }
    if (out->status) {
      L(k_gibbs_status, 1, 1, 256, 0, (const int*)cst, C, sst);
      put(out->status, sst, 1, 4, 1, 0);
    }
    if (ce != cudaSuccess) { cudaStreamSynchronize(h->stream); return fail(h, DFM_ERR_CUDA, "dfm_gibbs: copy failed"); }
    CK(cudaGetLastError());
  }
  CK(cudaStreamSynchronize(h->stream));
  return finish(h, mem);
}

int dfm_gibbs(dfm_handle* h, const double* X, const dfm_gibbs_opts* o, const dfm_em_init* init, const dfm_em_init* ref,
              const dfm_gibbs_out* out) {
  return gibbs_impl(h, X, o, init, ref, nullptr, out);
}

int dfm_gibbs_constrained(dfm_handle* h, const double* X, const dfm_gibbs_opts* o, const dfm_em_init* init, const dfm_em_init* ref,
                          const dfm_lam_constr* constr, const dfm_gibbs_out* out) {
  return gibbs_impl(h, X, o, init, ref, constr, out);
}

}  // extern "C"

// ------------------------------------------------------------------------------------ model batches
// dfm_series_responses, dfm_historical_decomposition, dfm_sign_restrictions, dfm_narrative_sign_restrictions and
// dfm_proxy_identification take n_model fitted models (dfm_em_init, back to back) and run over them in chunks of models, a size
// fixed by the shapes so that device memory does not grow with n_model.  ModelChunks reads the models a chunk at a time and runs
// the launches all of them start with; an OutSlot puts one output where the caller wants it.
namespace {

bool models_ok(const dfm_em_init* m) { return m && m->Lam && m->R && m->A && m->Q; }

// every model id below 2^40 (ids == nullptr: the ids are 0 .. n_model-1)
bool ids_ok(const unsigned long long* ids, int n_model) {
  for (int b = 0; ids && b < n_model; ++b)
    if (ids[b] >= (1ull << 40)) return false;
  return true;
}

// k_series_resp's plan for n_shock shocks to horizon H: hc horizons staged per pass (0: not even one fits), smR bytes of shared
// memory
struct SrPlan {
  int hc;
  size_t smR;
};
SrPlan series_resp_plan(int r, int n_shock, int H) {
  const size_t sm0 = series_resp_smem_doubles(r, n_shock, 0), rr = (size_t)r * r;
  const int hc = sm0 + rr > kMaxSmem / 8 ? 0 : (int)std::min<size_t>((size_t)H, (kMaxSmem / 8 - sm0) / rr);
  return {hc, series_resp_smem_doubles(r, n_shock, hc) * 8};
}

// Sign-restriction rows sorted by shock (stable): shock j's rows are off[j] .. off[j+1]-1; nj = the last restricted shock + 1
// (0-based), 0 without rows.  alloc and upload give the kernels their device copies.
struct SignRows {
  std::vector<int> series, horizon, sign, off;
  int nj = 0;
  int *d_series = nullptr, *d_horizon = nullptr, *d_sign = nullptr, *d_off = nullptr;
  void alloc(Arena& a) {
    d_off = a.get<int>(off.size());
    d_series = a.get<int>(series.size() + 1);
    d_horizon = a.get<int>(series.size() + 1);
    d_sign = a.get<int>(series.size() + 1);
  }
  int upload(dfm_handle* h) const {
    CK(cudaMemcpyAsync(d_off, off.data(), off.size() * sizeof(int), cudaMemcpyHostToDevice, h->stream));
    if (series.empty()) return DFM_OK;
    CK(cudaMemcpyAsync(d_series, series.data(), series.size() * sizeof(int), cudaMemcpyHostToDevice, h->stream));
    CK(cudaMemcpyAsync(d_horizon, horizon.data(), series.size() * sizeof(int), cudaMemcpyHostToDevice, h->stream));
    CK(cudaMemcpyAsync(d_sign, sign.data(), series.size() * sizeof(int), cudaMemcpyHostToDevice, h->stream));
    return DFM_OK;
  }
};

// rs's rows for n_shock shocks of N series to horizon H, range-checked (DFM_ERR_ARG with msg) and sorted into *s
int sign_rows(dfm_handle* h, const dfm_sign_restr* rs, int N, int H, int n_shock, const char* msg, SignRows* s) {
  for (int q = 0; q < rs->n; ++q)
    if (rs->series[q] < 0 || rs->series[q] >= N || rs->horizon[q] < 0 || rs->horizon[q] >= H || rs->shock[q] < 1 ||
        rs->shock[q] > n_shock || (rs->sign[q] != 1 && rs->sign[q] != -1))
      return fail(h, DFM_ERR_ARG, msg);
  s->off.assign(n_shock + 1, 0);
  for (int j = 1; j <= n_shock; ++j) {
    for (int q = 0; q < rs->n; ++q) {
      if (rs->shock[q] != j) continue;
      s->series.push_back(rs->series[q]);
      s->horizon.push_back(rs->horizon[q]);
      s->sign.push_back(rs->sign[q]);
      s->nj = j;
    }
    s->off[j] = (int)s->series.size();
  }
  return DFM_OK;
}

// The fitted models of a model-batch entry point, a chunk at a time.  alloc lays out, for B models: the staging of host inputs
// (Lam, R, A, Q, the Tp x r factor paths F when F is given, and scale), k_sr_prep's outputs, k_irf's when Hi > 0 (all r
// shocks to horizon Hi) and the chunk's model ids when with_ids (ids == nullptr: model j0 + b has id j0 + b).  Once per call
// setup uploads k_irf's shock list and scale; once per chunk, load points L_ .. F_ at the chunk's models (staged host arrays,
// or the caller's device arrays in place), uploads their ids and runs k_sr_prep, then k_irf.
struct ModelChunks {
  dfm_handle* h;
  const dfm_em_init* m;
  const double *F, *scale;
  const unsigned long long* ids;
  int N, r, p, Tp, Hi, mem;
  bool with_ids, hst;
  size_t Nr, rk, rr, kk, Tr;
  double *dL = nullptr, *dR = nullptr, *dA = nullptr, *dQ = nullptr, *dF = nullptr, *dS = nullptr;   // host-input staging
  double *M = nullptr, *Qs = nullptr, *G = nullptr, *irf = nullptr;  // k_sr_prep's (M, [I 0], [chol(Q); 0]) and k_irf's records
  int *st = nullptr, *shocks = nullptr;                               // per-model status, k_irf's shocks 0 .. r-1
  unsigned long long* dId = nullptr;
  std::vector<unsigned long long> hid;
  const double *L_ = nullptr, *R_ = nullptr, *A_ = nullptr, *Q_ = nullptr, *F_ = nullptr;   // the chunk's device views
  const double* sc = nullptr;                                                               // scale's (nullptr: 1)

  ModelChunks(dfm_handle* h, const dfm_em_init* m, int N, int r, int p, const double* scale, int mem, const double* F, int Tp,
              int Hi, bool with_ids, const unsigned long long* ids)
      : h(h), m(m), F(F), scale(scale), ids(ids), N(N), r(r), p(p), Tp(Tp), Hi(Hi), mem(mem), with_ids(with_ids),
        hst(mem == DFM_MEM_HOST), Nr((size_t)N * r), rk((size_t)r * r * p), rr((size_t)r * r),
        kk((size_t)r * p * r * p), Tr((size_t)Tp * r) {}

  void alloc(Arena& a, size_t B) {
    if (hst) {
      dL = a.get<double>(B * Nr);
      dR = a.get<double>(B * N);
      dA = a.get<double>(B * rk);
      dQ = a.get<double>(B * rr);
      dF = F ? a.get<double>(B * Tr) : nullptr;
      dS = scale ? a.get<double>(N) : nullptr;
    }
    M = a.get<double>(B * kk);
    Qs = a.get<double>(B * rk);
    G = a.get<double>(B * rk);
    st = a.get<int>(B);
    irf = Hi ? a.get<double>(B * rr * Hi) : nullptr;
    shocks = Hi ? a.get<int>(r) : nullptr;
    dId = with_ids ? a.get<unsigned long long>(B) : nullptr;
  }

  // Models per chunk: as many as kSimChunkBytes holds at layout(a, 1)'s bytes each (the 256-byte rounding and the buffers of
  // fixed size make that at least a B-model layout's bytes over B), at least one, at most cap.  layout(a, B) calls alloc(a, B)
  // and allocates the caller's own buffers.
  template <typename Lay> static int chunk_models(Lay&& layout, long long n_model, long long cap) {
    Arena a(nullptr);
    layout(a, 1);
    return (int)std::min<long long>({n_model, std::max<long long>(1, (long long)(kSimChunkBytes / a.off)), cap});
  }

  // grows the workspace to layout(a, B)'s bytes and lays the buffers out in it; uploads k_irf's shock list and scale
  template <typename Lay> int setup(Lay&& layout, size_t B) {
    CK(cudaSetDevice(h->device));
    int rc = lay_out(h, [&](Arena& a) { layout(a, B); });
    if (rc) return rc;
    if (Hi) {
      std::vector<int> all(r);
      for (int j = 0; j < r; ++j) all[j] = j;
      CK(cudaMemcpyAsync(shocks, all.data(), r * sizeof(int), cudaMemcpyHostToDevice, h->stream));
      DFM_SET_SMEM(k_irf, irf_smem_doubles(r * p) * 8);
    }
    sc = scale;
    if (hst && scale) {
      CK(cudaMemcpyAsync(dS, scale, (size_t)N * 8, cudaMemcpyHostToDevice, h->stream));
      sc = dS;
    }
    return DFM_OK;
  }

  int load(long long j0, int nm) {
    L_ = m->Lam + j0 * Nr;
    R_ = m->R + j0 * N;
    A_ = m->A + j0 * rk;
    Q_ = m->Q + j0 * rr;
    F_ = F ? F + j0 * Tr : nullptr;
    int rc = stage_in(h, L_, dL, nm * Nr, mem, &L_);
    if (!rc) rc = stage_in(h, R_, dR, nm * (size_t)N, mem, &R_);
    if (!rc) rc = stage_in(h, A_, dA, nm * rk, mem, &A_);
    if (!rc) rc = stage_in(h, Q_, dQ, nm * rr, mem, &Q_);
    if (!rc && F) rc = stage_in(h, F_, dF, nm * Tr, mem, &F_);
    if (rc) return rc;
    if (with_ids) {
      hid.resize(nm);
      for (int b = 0; b < nm; ++b) hid[b] = ids ? ids[j0 + b] : (unsigned long long)(j0 + b);
      CK(cudaMemcpyAsync(dId, hid.data(), nm * sizeof(unsigned long long), cudaMemcpyHostToDevice, h->stream));
    }
    L(k_sr_prep, nm, 1, 64, (rr + 8) * 8, A_, Q_, r, p, M, Qs, G, st);
    if (Hi)
      L(k_irf, r, nm, 64, irf_smem_doubles(r * p) * 8, (const double*)M, (const double*)Qs, (const double*)G, r * p, r, Hi, r,
        (const int*)shocks, irf);
    return DFM_OK;
  }

  // body(j0, nm) on each chunk of nb models, after load(j0, nm).  On the host path the stream is synchronised at the end of each
  // chunk, because the next one reuses the staging buffers.
  template <typename Body> int run(long long n_model, int nb, Body&& body) {
    for (long long j0 = 0; j0 < n_model; j0 += nb) {
      const int nm = (int)std::min<long long>(nb, n_model - j0);
      int rc = load(j0, nm);
      if (!rc) rc = body(j0, nm);
      if (rc) return rc;
      if (hst) CK(cudaStreamSynchronize(h->stream));
    }
    return finish(h, mem);
  }

  // the copy-back of the nm models from j0 of every slot, up to the first error
  template <typename... T> int flush(long long j0, long long nm, const OutSlot<T>&... s) const {
    return ::flush(h, j0, nm, mem, s...);
  }
};

}  // namespace

extern "C" {

// ------------------------------------------------------------------------------------ series responses / FEVD
// Per chunk of models (ModelChunks): k_sr_prep -> k_irf (all r shocks) -> k_series_resp.
int dfm_series_responses(dfm_handle* h, const dfm_em_init* models, int N, int r, int p, int n_model, int H, int n_shock,
                         const double* scale, int mem, double* resp, double* fevd, int* status) {
  if (!h || !models_ok(models) || N <= 0 || r <= 0 || r > 64 || p <= 0 || n_model <= 0 || H <= 0 || n_shock <= 0 || n_shock > r ||
      (mem != DFM_MEM_HOST && mem != DFM_MEM_DEVICE))
    return fail(h, DFM_ERR_ARG, "dfm_series_responses: bad argument");
  const SrPlan sp = series_resp_plan(r, n_shock, H);
  if (!sp.hc) return fail(h, DFM_ERR_UNSUPPORTED, "dfm_series_responses: r too large");
  if (irf_smem_doubles(r * p) * 8 > kMaxSmem)
    return fail(h, DFM_ERR_UNSUPPORTED, "dfm_series_responses: state dimension r*p too large (r*p > 14076)");
  const bool hst = mem == DFM_MEM_HOST;
  const size_t nout = (size_t)N * H * n_shock;
  ModelChunks mc(h, models, N, r, p, scale, mem, nullptr, 0, H, false, nullptr);
  OutSlot<double> oRe, oFe;
  auto layout = [&](Arena& a, size_t B) {
    mc.alloc(a, B);
    oRe = staged(a, resp, nout, B, hst);
    oFe = staged(a, fevd, nout, B, hst);
  };
  const int nb = ModelChunks::chunk_models(layout, n_model, kMaxGridBatch);
  int rc = mc.setup(layout, nb);
  if (rc) return rc;
  DFM_SET_SMEM(k_series_resp, sp.smR);
  const OutSlot<int> ost{status, mc.st, 1};
  return mc.run(n_model, nb, [&](long long j0, int nm) {
    L(k_series_resp, (N + SR_NS - 1) / SR_NS, nm, SR_NS, sp.smR, mc.L_, mc.R_, mc.sc, (const double*)mc.irf, (const int*)mc.st, N, r, H,
      n_shock, sp.hc, 1, oRe.at(j0), oFe.at(j0));
    return mc.flush(j0, nm, oRe, oFe, ost);
  });
}

// ------------------------------------------------------------------------------------ historical decompositions
// Per chunk of models (ModelChunks): k_sr_prep -> k_hd_paths -> k_hd_series.  The shocks are written to scratch when they are not
// asked for.
int dfm_historical_decomposition(dfm_handle* h, const dfm_em_init* models, const double* F, const double* scale,
                                 const dfm_hd_opts* o, const dfm_hd_out* out) {
  if (!h || !models_ok(models) || !F || !o || !out || o->N <= 0 || o->r <= 0 || o->p <= 0 || o->Tp <= 0 || o->n_model <= 0 ||
      o->t0 < o->p - 1 || o->t0 >= o->Tp || o->n_shock < 1 || o->n_shock > o->r || (o->mem != DFM_MEM_HOST && o->mem != DFM_MEM_DEVICE))
    return fail(h, DFM_ERR_ARG, "dfm_historical_decomposition: bad argument");
  const int N = o->N, r = o->r, p = o->p, Tp = o->Tp, ns = o->n_shock, nc = ns + 2, mem = o->mem;
  if (r * p > 48) return fail(h, DFM_ERR_UNSUPPORTED, "dfm_historical_decomposition: state dimension r*p > 48");
  const size_t Tr = (size_t)Tp * r, nY = (size_t)nc * Tr, nC = (size_t)N * Tp * ns, nB = (size_t)N * Tp;
  const size_t smP = hd_paths_smem_doubles(r, p, nc) * 8;
  // rows of the recursions staged per pass of k_hd_series: about 16 KB of shared memory in all (at least one row), so that many
  // CTAs share an SM
  const size_t budget = std::max<size_t>(2048, (size_t)r * HD_NS + (size_t)nc * r);
  const int tc = (int)std::min<size_t>((size_t)Tp, (budget - (size_t)r * HD_NS) / ((size_t)nc * r));
  const size_t smS = hd_series_smem_doubles(r, nc, tc) * 8;
  const bool hst = mem == DFM_MEM_HOST;
  ModelChunks mc(h, models, N, r, p, scale, mem, F, Tp, 0, false, nullptr);
  OutSlot<double> oE, oC, oR, oB;
  double* dY = nullptr;
  auto layout = [&](Arena& a, size_t B) {
    mc.alloc(a, B);
    oE = scratch(a, out->shocks, Tr, B, hst);
    oC = staged(a, out->contrib, nC, B, hst);
    oR = staged(a, out->rest, nB, B, hst);
    oB = staged(a, out->base, nB, B, hst);
    dY = a.get<double>(B * nY);
  };
  const int nb = ModelChunks::chunk_models(layout, o->n_model, kMaxGridBatch);
  int rc = mc.setup(layout, nb);
  if (rc) return rc;
  DFM_SET_SMEM(k_hd_paths, smP);
  const OutSlot<int> ost{out->status, mc.st, 1};
  // k_hd_series holds each series' loadings in RM >= r registers
  auto series = [&](auto rm, long long j0, int nm) {
    constexpr int RM = decltype(rm)::value;
    DFM_SET_SMEM(k_hd_series<RM>, smS);
    L(k_hd_series<RM>, (N + HD_NS - 1) / HD_NS, nm, HD_NS, smS, mc.L_, mc.R_, mc.sc, (const double*)dY, (const int*)mc.st, N, r, Tp, ns,
      tc, oC.at(j0), oR.at(j0), oB.at(j0));
  };
  return mc.run(o->n_model, nb, [&](long long j0, int nm) {
    L(k_hd_paths, nm, 1, HD_PT, smP, (const double*)mc.M, (const double*)mc.G, mc.F_, r, p, Tp, o->t0, ns, mc.st, oE.at(j0), dY);
    if (r <= 8) series(std::integral_constant<int, 8>(), j0, nm);
    else if (r <= 16) series(std::integral_constant<int, 16>(), j0, nm);
    else if (r <= 32) series(std::integral_constant<int, 32>(), j0, nm);
    else series(std::integral_constant<int, 48>(), j0, nm);
    return mc.flush(j0, nm, oE, oC, oR, oB, ost);
  });
}

// ------------------------------------------------------------------------------------ sign restrictions
// Per chunk of models (ModelChunks; at most 65 535 rotated records): k_sr_prep -> k_irf (all r shocks) -> k_sign_prep -> per batch
// of candidates (a size fixed by n_rot) k_sign_cand -> k_sign_pick -> k_sign_rot -> k_series_resp on the n_keep rotated records
// of every model.
int dfm_sign_restrictions(dfm_handle* h, const dfm_em_init* models, const unsigned long long* ids, const double* scale,
                          const dfm_sign_opts* o, const dfm_sign_restr* rs, const dfm_sign_out* out) {
  if (!h || !models_ok(models) || !o || !rs || !out || o->N <= 0 || o->r <= 0 || o->p <= 0 || o->n_model <= 0 || o->H <= 0 ||
      o->n_shock < 1 || o->n_shock > o->r || o->n_rot < 1 || o->n_keep < 1 || rs->n < 0 ||
      (rs->n > 0 && (!rs->series || !rs->horizon || !rs->shock || !rs->sign)) || (o->mem != DFM_MEM_HOST && o->mem != DFM_MEM_DEVICE))
    return fail(h, DFM_ERR_ARG, "dfm_sign_restrictions: bad argument");
  const int N = o->N, r = o->r, p = o->p, H = o->H, ns = o->n_shock, nR = rs->n, nk = o->n_keep, mem = o->mem;
  SignRows sr;
  int rc = sign_rows(h, rs, N, H, ns, "dfm_sign_restrictions: a restriction row outside its range", &sr);
  if (rc) return rc;
  if (!ids_ok(ids, o->n_model)) return fail(h, DFM_ERR_ARG, "dfm_sign_restrictions: a model id >= 2^40");
  if (r > SG_RMAX || nR > SG_NRMAX || r * p > 48 || nk > kMaxGridBatch)
    return fail(h, DFM_ERR_UNSUPPORTED, "dfm_sign_restrictions: r > 16, more than 256 rows, r*p > 48 or n_keep > 65535");
  const int nj = sr.nj;
  const size_t rr = (size_t)r * r, nout = (size_t)N * H * ns;
  const SrPlan sp = series_resp_plan(r, ns, H);
  const size_t smC = sign_cand_smem_bytes(r, nj, nR), smT = sign_rot_smem_bytes(r, nj, nR);
  // candidates per model and batch: whole CTAs of SG_NT, at most 2^20
  const long long nct = std::min<long long>((o->n_rot + SG_NT - 1) / SG_NT, (1LL << 20) / SG_NT);
  const int ntile = (int)(nct * (SG_NT / SG_TILE));
  const bool hst = mem == DFM_MEM_HOST;
  ModelChunks mc(h, models, N, r, p, scale, mem, nullptr, 0, H, true, ids);
  OutSlot<double> oRo, oRe, oFe;
  double *dC = nullptr, *dRec = nullptr;
  long long *dNa = nullptr, *dCa = nullptr;
  unsigned* dMask = nullptr;
  int* dSst = nullptr;
  auto layout = [&](Arena& a, size_t B) {
    mc.alloc(a, B);
    sr.alloc(a);
    oRo = staged(a, out->rot, nk * rr, B, hst);
    oRe = staged(a, out->resp, nk * nout, B, hst);
    oFe = staged(a, out->fevd, nk * nout, B, hst);
    dC = a.get<double>(B * nR * r + 1);
    dRec = a.get<double>(B * nk * rr * H);
    dNa = a.get<long long>(B);
    dCa = a.get<long long>(B * nk);
    dMask = a.get<unsigned>(B * ntile);
    dSst = a.get<int>(B * nk);
  };
  const int nb = ModelChunks::chunk_models(layout, o->n_model, kMaxGridBatch / nk);
  rc = mc.setup(layout, nb);
  if (!rc) rc = sr.upload(h);
  if (rc) return rc;
  DFM_SET_SMEM(k_series_resp, sp.smR);
  DFM_SET_SMEM(k_sign_cand, smC);
  DFM_SET_SMEM(k_sign_rot, smT);
  const OutSlot<long long> ona{out->n_accept, dNa, 1}, oca{out->cand, dCa, (size_t)nk};
  const OutSlot<int> ost{out->status, mc.st, 1};
  return mc.run(o->n_model, nb, [&](long long j0, int nm) {
    double *oRe_ = oRe.at(j0), *oFe_ = oFe.at(j0);
    L(k_sign_prep, nm, 1, 64, 8, mc.L_, mc.R_, (const double*)mc.irf, N, r, H, nR, (const int*)sr.d_series, (const int*)sr.d_horizon,
      (const int*)sr.d_sign, nk, mc.st, dC, dNa, dCa);
    for (long long c0 = 0; c0 < o->n_rot; c0 += (long long)ntile * SG_TILE) {
      L(k_sign_cand, ntile / (SG_NT / SG_TILE), nm, SG_NT, smC, (const double*)dC, (const int*)sr.d_off, (const int*)mc.st, r, nR, nj,
        c0, o->n_rot, ntile, o->seed, (const unsigned long long*)mc.dId, dMask);
      L(k_sign_pick, nm, 1, SG_PT, 2 * SG_PT * sizeof(int), (const unsigned*)dMask, ntile, c0, nk, (const int*)mc.st, dNa, dCa);
    }
    L(k_sign_rot, nm * nk, 1, 64, smT, (const double*)mc.irf, (const double*)dC, (const int*)sr.d_off, (const int*)mc.st,
      (const long long*)dCa, r, H, nR, nj, nk, o->seed, (const unsigned long long*)mc.dId, oRo.at(j0), dRec, dSst);
    if (oRe_ || oFe_)
      L(k_series_resp, (N + SR_NS - 1) / SR_NS, nm * nk, SR_NS, sp.smR, mc.L_, mc.R_, mc.sc, (const double*)dRec, (const int*)dSst, N,
        r, H, ns, sp.hc, nk, oRe_, oFe_);
    return mc.flush(j0, nm, oRo, oRe, oFe, ona, oca, ost);
  });
}

// ------------------------------------------------------------------------------------ narrative sign restrictions
// dfm_sign_restrictions' pipeline with k_narr_prep after k_sign_prep, k_narr_cand / k_narr_rot in place of k_sign_cand /
// k_sign_rot, and k_narr_omega -> k_narr_weight on the kept slots.  The narrative rows are sorted as the kernels read them:
// kinds 0 and 3 by shock (stable), then kinds 1 and 2.
int dfm_narrative_sign_restrictions(dfm_handle* h, const dfm_em_init* models, const double* F, const unsigned long long* ids,
                                    const double* scale, const dfm_narr_opts* o, const dfm_sign_restr* rs, const dfm_narr_restr* nr,
                                    const dfm_narr_out* out) {
  if (!h || !models_ok(models) || !F || !o || !rs || !nr || !out || o->N <= 0 || o->r <= 0 || o->p <= 0 || o->n_model <= 0 ||
      o->H <= 0 || o->n_shock < 1 || o->n_shock > o->r || o->n_rot < 1 || o->n_keep < 1 || o->Tp < 1 || o->n_sim < 1 || rs->n < 0 ||
      (rs->n > 0 && (!rs->series || !rs->horizon || !rs->shock || !rs->sign)) || nr->n < 0 ||
      (nr->n > 0 && (!nr->kind || !nr->shock || !nr->series || !nr->row || !nr->h || !nr->sign)) ||
      (o->mem != DFM_MEM_HOST && o->mem != DFM_MEM_DEVICE))
    return fail(h, DFM_ERR_ARG, "dfm_narrative_sign_restrictions: bad argument");
  const int N = o->N, r = o->r, p = o->p, H = o->H, ns = o->n_shock, nR = rs->n, nN = nr->n, nk = o->n_keep, Tp = o->Tp, mem = o->mem;
  SignRows sr;
  int rc = sign_rows(h, rs, N, H, ns, "dfm_narrative_sign_restrictions: a restriction row outside its range", &sr);
  if (rc) return rc;
  for (int q = 0; q < nN; ++q) {
    const int kd = nr->kind[q], hh = kd == 0 ? 0 : nr->h[q];
    if (kd < 0 || kd > 3 || nr->shock[q] < 1 || nr->shock[q] > ns || ((kd == 0 || kd == 3) && nr->sign[q] != 1 && nr->sign[q] != -1) ||
        (kd != 0 && (nr->series[q] < 0 || nr->series[q] >= N)) || nr->row[q] < p || hh < 0 || hh >= H || nr->row[q] + hh >= Tp)
      return fail(h, DFM_ERR_ARG, "dfm_narrative_sign_restrictions: a narrative row outside its range");
  }
  if (!ids_ok(ids, o->n_model)) return fail(h, DFM_ERR_ARG, "dfm_narrative_sign_restrictions: a model id >= 2^40");
  if (r > SG_RMAX || nR > SG_NRMAX || r * p > 48 || nk > kMaxGridBatch || nN > NR_NMAX || o->n_sim > (1 << 20))
    return fail(h, DFM_ERR_UNSUPPORTED, "dfm_narrative_sign_restrictions: r > 16, more than 256 sign rows or 64 narrative rows, "
                                        "r*p > 48, n_keep > 65535 or n_sim > 2^20");
  // the periods' union (positions), the narrative rows in the kernels' order
  std::vector<char> inP(Tp, 0);
  for (int q = 0; q < nN; ++q) for (int t = nr->row[q]; t <= nr->row[q] + (nr->kind[q] == 0 ? 0 : nr->h[q]); ++t) inP[t] = 1;
  std::vector<int> pos(Tp, 0);
  int nP = 0;
  for (int t = 0; t < Tp; ++t) { pos[t] = nP; nP += inP[t]; }
  if ((long long)nP * r > (1 << 14)) return fail(h, DFM_ERR_UNSUPPORTED, "dfm_narrative_sign_restrictions: nP * r > 2^14");
  std::vector<int> noff(ns + 1, 0);
  std::vector<nr_row> rows;
  int nT = sr.nj, nD = 0, nC = 0;
  auto add = [&](int q) {
    nr_row w;
    w.kind = nr->kind[q]; w.shock = nr->shock[q] - 1; w.series = w.kind == 0 ? 0 : nr->series[q]; w.t = nr->row[q];
    w.h = w.kind == 0 ? 0 : nr->h[q]; w.sign = (w.kind == 1 || w.kind == 2) ? 1 : nr->sign[q];
    w.doff = nD; nD += w.kind == 0 ? r : r * r;
    w.pos = pos[w.t];
    w.coff = nC; if (w.kind != 0) nC += (w.h + 1) * r;
    rows.push_back(w);
  };
  for (int j = 1; j <= ns; ++j) {
    for (int q = 0; q < nN; ++q)
      if (nr->shock[q] == j && (nr->kind[q] == 0 || nr->kind[q] == 3)) { add(q); nT = std::max(nT, j); }
    noff[j] = (int)rows.size();
  }
  for (int q = 0; q < nN; ++q) if (nr->kind[q] == 1 || nr->kind[q] == 2) add(q);
  const bool share = (int)rows.size() > noff[ns];
  sr.off.resize(nT + 1); noff.resize(nT + 1);
  const int ncol = share ? r : nT;
  const size_t smC = narr_cand_smem_bytes(ncol, r, nT, nR, nD, nN), smT = narr_rot_smem_bytes(r, nT, nR, nD, nN);
  const size_t smO = (size_t)nC * 8 + 8;
  if (smC > kMaxSmem || smO > kMaxSmem)
    return fail(h, DFM_ERR_UNSUPPORTED, "dfm_narrative_sign_restrictions: the rows do not fit the kernels' shared memory");
  const size_t rk = (size_t)r * r * p, rr = (size_t)r * r, nout = (size_t)N * H * ns, Tr = (size_t)Tp * r, nE = (size_t)Tp * ns;
  const SrPlan sp = series_resp_plan(r, ns, H);
  const size_t smP = (rk + rr + 1) * 8;
  const long long nct = std::min<long long>((o->n_rot + SG_NT - 1) / SG_NT, (1LL << 20) / SG_NT);
  const int ntile = (int)(nct * (SG_NT / SG_TILE));
  const int ntl = (o->n_sim + NR_SIMT - 1) / NR_SIMT;
  const bool hst = mem == DFM_MEM_HOST;
  ModelChunks mc(h, models, N, r, p, scale, mem, F, Tp, H, true, ids);
  OutSlot<double> oRo, oRe, oFe, oEp, oW;
  OutSlot<long long> oNo;
  double *dC = nullptr, *dRec = nullptr, *dU = nullptr, *dD = nullptr;
  long long *dNa = nullptr, *dCa = nullptr;
  unsigned long long* dNok = nullptr;
  unsigned* dMask = nullptr;
  int *dSst = nullptr, *dNoff = nullptr;
  nr_row* dRows = nullptr;
  auto layout = [&](Arena& a, size_t B) {
    mc.alloc(a, B);
    sr.alloc(a);
    oRo = staged(a, out->rot, nk * rr, B, hst);
    oRe = staged(a, out->resp, nk * nout, B, hst);
    oFe = staged(a, out->fevd, nk * nout, B, hst);
    oEp = staged(a, out->eps, nk * nE, B, hst);
    oW = staged(a, out->weight, (size_t)nk, B, hst);
    oNo = staged(a, out->n_ok, (size_t)nk, B, hst);
    dC = a.get<double>(B * nR * r + 1);
    dRec = a.get<double>(B * nk * rr * H);
    dU = a.get<double>(B * Tr);
    dD = a.get<double>(B * nD + 1);
    dNa = a.get<long long>(B);
    dCa = a.get<long long>(B * nk);
    dNok = a.get<unsigned long long>(B * nk);
    dMask = a.get<unsigned>(B * ntile);
    dSst = a.get<int>(B * nk);
    dNoff = a.get<int>(nT + 1);
    dRows = a.get<nr_row>(nN + 1);
  };
  const int nb = ModelChunks::chunk_models(layout, o->n_model, kMaxGridBatch / nk);
  rc = mc.setup(layout, nb);
  if (!rc) rc = sr.upload(h);
  if (rc) return rc;
  CK(cudaMemcpyAsync(dNoff, noff.data(), (nT + 1) * sizeof(int), cudaMemcpyHostToDevice, h->stream));
  if (nN) CK(cudaMemcpyAsync(dRows, rows.data(), nN * sizeof(nr_row), cudaMemcpyHostToDevice, h->stream));
  DFM_SET_SMEM(k_series_resp, sp.smR);
  DFM_SET_SMEM(k_narr_cand, smC);
  DFM_SET_SMEM(k_narr_rot, smT);
  DFM_SET_SMEM(k_narr_omega, smO);
  const OutSlot<long long> ona{out->n_accept, dNa, 1}, oca{out->cand, dCa, (size_t)nk};
  const OutSlot<int> ost{out->status, mc.st, 1};
  return mc.run(o->n_model, nb, [&](long long j0, int nm) -> int {
    const size_t S = (size_t)nm * nk;
    double *oRe_ = oRe.at(j0), *oFe_ = oFe.at(j0), *oEp_ = oEp.at(j0), *oW_ = oW.at(j0);
    long long* oNo_ = oNo.at(j0);
    L(k_sign_prep, nm, 1, 64, 8, mc.L_, mc.R_, (const double*)mc.irf, N, r, H, nR, (const int*)sr.d_series, (const int*)sr.d_horizon,
      (const int*)sr.d_sign, nk, mc.st, dC, dNa, dCa);
    L(k_narr_prep, nm, 1, NR_PT, smP, mc.L_, mc.R_, (const double*)mc.irf, (const double*)mc.M, (const double*)mc.G, mc.F_, N, r, p, H,
      Tp, nN, (const nr_row*)dRows, nD, mc.st, dU, dD);
    for (long long c0 = 0; c0 < o->n_rot; c0 += (long long)ntile * SG_TILE) {
      L(k_narr_cand, ntile / (SG_NT / SG_TILE), nm, SG_NT, smC, (const double*)dC, (const int*)sr.d_off, (const double*)dD,
        (const nr_row*)dRows, (const int*)dNoff, (const int*)mc.st, r, nR, nD, nN, nT, ncol, c0, o->n_rot, ntile, o->seed,
        (const unsigned long long*)mc.dId, dMask);
      L(k_sign_pick, nm, 1, SG_PT, 2 * SG_PT * sizeof(int), (const unsigned*)dMask, ntile, c0, nk, (const int*)mc.st, dNa, dCa);
    }
    L(k_narr_rot, nm * nk, 1, 64, smT, (const double*)mc.irf, (const double*)dC, (const int*)sr.d_off, (const double*)dD,
      (const nr_row*)dRows, (const int*)dNoff, (const double*)dU, (const int*)mc.st, (const long long*)dCa, r, H, Tp, nR, nD, nN, nT,
      nk, oEp_ ? ns : 0, o->seed, (const unsigned long long*)mc.dId, oRo.at(j0), dRec, dSst, oEp_, dNok);
    if (oRe_ || oFe_)
      L(k_series_resp, (N + SR_NS - 1) / SR_NS, nm * nk, SR_NS, sp.smR, mc.L_, mc.R_, mc.sc, (const double*)dRec, (const int*)dSst, N,
        r, H, ns, sp.hc, nk, oRe_, oFe_);
    if (nN && (oW_ || oNo_))
      L(k_narr_omega, nm * nk, ntl, NR_SIMT, smO, mc.L_, (const double*)dRec, (const nr_row*)dRows, (const int*)dSst,
        (const unsigned long long*)mc.dId, N, r, H, nN, nC, nP, o->n_sim, nk, o->seed, dNok);
    if (oW_ || oNo_) {
      if (!nN) {                                         // no narrative rows: every simulation satisfies them
        std::vector<unsigned long long> all(S, (unsigned long long)o->n_sim);
        CK(cudaMemcpyAsync(dNok, all.data(), S * sizeof(unsigned long long), cudaMemcpyHostToDevice, h->stream));
        CK(cudaStreamSynchronize(h->stream));
      }
      L(k_narr_weight, (int)((S + NR_PT - 1) / NR_PT), 1, NR_PT, 0, (const unsigned long long*)dNok, (const int*)dSst, (int)S, o->n_sim,
        oNo_, oW_);
    }
    return mc.flush(j0, nm, oRo, oRe, oFe, oEp, oW, oNo, ona, oca, ost);
  });
}

// ------------------------------------------------------------------------------------ proxy (external instrument) identification
// Per chunk of models (ModelChunks): k_sr_prep -> k_irf (when responses are asked for) -> k_iv_prep -> k_iv_boot -> per batch of
// records (model, instrument, replicate) in output order: k_iv_rot -> k_series_resp (n_shock 1).  A chunk holds several models
// when all their records fit one batch, otherwise one model whose records run in several batches; either way record s of a batch
// reads model s / (n_inst (1 + n_boot)) of the chunk.  omega is written to scratch when it is not asked for.
int dfm_proxy_identification(dfm_handle* h, const dfm_em_init* models, const double* F, const double* Z, const unsigned long long* ids,
                             const double* scale, const dfm_proxy_opts* o, const dfm_proxy_out* out) {
  if (!h || !models_ok(models) || !F || !Z || !o || !out || o->N <= 0 || o->r <= 0 || o->p <= 0 || o->n_model <= 0 || o->Tp < 1 ||
      o->H <= 0 || o->n_inst < 1 || o->i0 < 0 || o->i0 >= o->N || o->q < 0 || o->block < 1 || o->n_boot < 0 ||
      (o->mem != DFM_MEM_HOST && o->mem != DFM_MEM_DEVICE))
    return fail(h, DFM_ERR_ARG, "dfm_proxy_identification: bad argument");
  if (!ids_ok(ids, o->n_model)) return fail(h, DFM_ERR_ARG, "dfm_proxy_identification: a model id >= 2^40");
  const int N = o->N, r = o->r, p = o->p, H = o->H, Tp = o->Tp, ni = o->n_inst, nbt = o->n_boot, mem = o->mem;
  if (r * p > 48 || ni > IV_NIMAX || nbt > 65535)
    return fail(h, DFM_ERR_UNSUPPORTED, "dfm_proxy_identification: r*p > 48, n_inst > 8 or n_boot > 65535");
  const size_t smP = iv_prep_smem_bytes(r, Tp), smB = iv_boot_smem_bytes(r, Tp), smT = iv_rot_smem_bytes(r);
  if (smP > kMaxSmem || smB > kMaxSmem)
    return fail(h, DFM_ERR_UNSUPPORTED, "dfm_proxy_identification: Tp (r + 1) + 64 r > 28160 (the bootstrap's shared memory)");
  const bool want = out->resp || out->fevd, hst = mem == DFM_MEM_HOST;
  const size_t rr = (size_t)r * r, Tr = (size_t)Tp * r, NH = (size_t)N * H, P = (size_t)ni * (nbt + 1), nE = (size_t)ni * Tp;
  const SrPlan sp = series_resp_plan(r, 1, H);
  ModelChunks mc(h, models, N, r, p, scale, mem, F, Tp, want ? H : 0, true, ids);
  OutSlot<double> oOm, oEp, oRel, oPi, oFs, oRe, oFe;
  OutSlot<int> oNo;
  double *dZ = nullptr, *dU = nullptr, *dRec = nullptr;
  int *dIdx = nullptr, *dNk = nullptr, *dIst = nullptr, *dSst = nullptr;
  // B models and R records (responses and their staging)
  auto layout = [&](Arena& a, size_t B, size_t R) {
    mc.alloc(a, B);
    dZ = hst ? a.get<double>(nE) : nullptr;
    oOm = scratch(a, out->omega, P * r, B, hst);
    oEp = staged(a, out->eps, nE, B, hst);
    oRel = staged(a, out->reliability, (size_t)ni, B, hst);
    oPi = staged(a, out->fs_pi, (size_t)ni, B, hst);
    oFs = staged(a, out->fs_F, (size_t)ni, B, hst);
    oNo = staged(a, out->n_obs, (size_t)ni, B, hst);
    dU = a.get<double>(B * Tr);
    dIdx = a.get<int>(B * nE);
    dNk = a.get<int>(B * ni);
    dIst = a.get<int>(B * ni);
    oRe = staged(a, out->resp, NH, R, hst);
    oFe = staged(a, out->fevd, NH, R, hst);
    dRec = a.get<double>(R * rr * H);
    dSst = a.get<int>(R);
  };
  auto bytes = [&](size_t B, size_t R) {
    Arena a(nullptr);
    layout(a, B, R);
    return a.off;
  };
  // records per batch: grid.y of k_series_resp, and half of kSimChunkBytes; models per chunk: the other half, grid.y of k_iv_boot,
  // and (for more than one) all their records in one batch
  const long long cap = std::min<long long>(kMaxGridBatch, std::max<long long>(1, (long long)(kSimChunkBytes / 2 / bytes(0, 1))));
  const int nb = (int)std::max<long long>(1, std::min<long long>({(long long)o->n_model, (long long)(kSimChunkBytes / 2 / bytes(1, 0)),
                                                                  (long long)(kMaxGridBatch / ni), cap / (long long)P}));
  const long long nrec = std::min<long long>(cap, (long long)nb * (long long)P);
  int rc = mc.setup([&](Arena& a, size_t B) { layout(a, B, want ? nrec : 0); }, nb);
  if (rc) return rc;
  const double* Z_ = Z;
  rc = stage_in(h, Z, dZ, nE, mem, &Z_);
  if (rc) return rc;
  DFM_SET_SMEM(k_series_resp, sp.smR);
  DFM_SET_SMEM(k_iv_prep, smP);
  DFM_SET_SMEM(k_iv_boot, smB);
  const OutSlot<int> ost{out->status, dIst, (size_t)ni};
  return mc.run(o->n_model, nb, [&](long long j0, int nm) -> int {
    double* oOm_ = oOm.at(j0);
    L(k_iv_prep, nm, 1, IV_PT, smP, mc.L_, mc.R_, mc.A_, (const double*)mc.G, mc.F_, Z_, N, r, p, Tp, ni, o->i0, o->q, nbt,
      (const int*)mc.st, dU, dIdx, dNk, dIst, oOm_, oEp.at(j0), oNo.at(j0), oRel.at(j0), oPi.at(j0), oFs.at(j0));
    if (nbt > 0)
      L(k_iv_boot, (nbt + IV_BT - 1) / IV_BT, nm * ni, IV_BT, smB, (const double*)dU, Z_, (const int*)dIdx, (const int*)dNk,
        (const int*)dIst, r, Tp, ni, o->block, nbt, o->seed, (const unsigned long long*)mc.dId, oOm_);
    const long long nrc = (long long)nm * (long long)P;
    for (long long g0 = 0; want && g0 < nrc; g0 += nrec) {
      const int nr = (int)std::min<long long>(nrec, nrc - g0);
      const long long s0 = j0 * (long long)P + g0;           // the batch's first record in the outputs
      L(k_iv_rot, nr, 1, 64, smT, (const double*)mc.irf, (const double*)oOm_, g0, r, H, ni, nbt, dRec, dSst);
      L(k_series_resp, (N + SR_NS - 1) / SR_NS, nr, SR_NS, sp.smR, mc.L_, mc.R_, mc.sc, (const double*)dRec, (const int*)dSst, N, r, H, 1,
        sp.hc, (int)P, oRe.at(s0), oFe.at(s0));
      if (int e = mc.flush(s0, nr, oRe, oFe)) return e;
      if (hst) CK(cudaStreamSynchronize(h->stream));         // (the next batch rewrites the staging of resp and fevd)
    }
    return mc.flush(j0, nm, oOm, oEp, oRel, oPi, oFs, oNo, ost);
  });
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
  double *dD, *dF, *dc, *dq, *dq0;
  int* dst;
  int rc = lay_out(h, [&](Arena& a) {
    dD = mem == DFM_MEM_HOST ? a.get<double>((size_t)T * ns) : nullptr;
    dF = mem == DFM_MEM_HOST ? a.get<double>((size_t)T * r) : nullptr;
    dc = a.get<double>(ns); dq = a.get<double>(ns); dq0 = a.get<double>(ns); dst = a.get<int>(ns);
  });
  if (rc) return rc;
  const double *x, *f;
  rc = stage_in(h, data, dD, (size_t)T * ns, mem, &x); if (rc) return rc;
  rc = stage_in(h, F, dF, (size_t)T * r, mem, &f); if (rc) return rc;
  CK(cudaMemsetAsync(dst, 0, ns * sizeof(int), h->stream));
  DFM_SET_SMEM(k_instability, smem);
  L(k_instability, ns, 1, 256, smem, x, f, T, ns, r, q, T_break, ccut, min_obs, dc, dq, qlr0 ? dq0 : (double*)nullptr, dst);
  rc = copy_out(h, chow, dc, ns, mem); if (rc) return rc;
  rc = copy_out(h, qlr, dq, ns, mem); if (rc) return rc;
  if (qlr0) { rc = copy_out(h, qlr0, dq0, ns, mem); if (rc) return rc; }
  if (status) { rc = copy_out(h, status, dst, ns, mem); if (rc) return rc; }
  return finish(h, mem);
}

int dfm_fit_correlation(dfm_handle* h, const double* data, const double* F, const double* F_alt, int T, int ns, int r, int T_break,
                        int min_obs, int mem, double* cor, int* status) {
  if (!h || !data || !F || !F_alt || !cor || T <= 2 || ns <= 0 || r <= 0 || r > 48 || T_break <= 0 || T_break >= T || min_obs < 0)
    return fail(h, DFM_ERR_ARG, "dfm_fit_correlation: bad argument");
  CK(cudaSetDevice(h->device));
  double *dD, *dF, *dFa, *dc;
  int* dst;
  int rc = lay_out(h, [&](Arena& a) {
    dD = mem == DFM_MEM_HOST ? a.get<double>((size_t)T * ns) : nullptr;
    dF = mem == DFM_MEM_HOST ? a.get<double>((size_t)T * r) : nullptr;
    dFa = mem == DFM_MEM_HOST ? a.get<double>((size_t)T * r) : nullptr;
    dc = a.get<double>(ns); dst = a.get<int>(ns);
  });
  if (rc) return rc;
  const double *x, *f, *fa;
  rc = stage_in(h, data, dD, (size_t)T * ns, mem, &x); if (rc) return rc;
  rc = stage_in(h, F, dF, (size_t)T * r, mem, &f); if (rc) return rc;
  rc = stage_in(h, F_alt, dFa, (size_t)T * r, mem, &fa); if (rc) return rc;
  CK(cudaMemsetAsync(dst, 0, ns * sizeof(int), h->stream));
  L(k_fit_corr, ns, 1, 128, (size_t)(2 * (r * r + 2 * r) + 64 + 48 + 8) * 8, x, f, fa, T, ns, r, T_break, min_obs, dc, dst);
  rc = copy_out(h, cor, dc, ns, mem); if (rc) return rc;
  if (status) { rc = copy_out(h, status, dst, ns, mem); if (rc) return rc; }
  return finish(h, mem);
}

int dfm_percentiles(dfm_handle* h, const double* recs, long long n, int d, const double* q, int nq, int mem, double* out) {
  if (!h || !recs || !q || !out || n <= 0 || d <= 0 || nq <= 0 || nq > 64) return fail(h, DFM_ERR_ARG, "dfm_percentiles: bad argument");
  for (int k = 0; k < nq; ++k) if (!(q[k] >= 0.0 && q[k] <= 100.0)) return fail(h, DFM_ERR_ARG, "dfm_percentiles: q outside [0, 100]");
  long long npad = 2; while (npad < n) npad <<= 1;
  size_t smem = (size_t)(npad + 2) * 8;
  if (smem > kMaxSmem) return fail(h, DFM_ERR_UNSUPPORTED, "dfm_percentiles: more than 16384 replications");
  CK(cudaSetDevice(h->device));
  const bool hst = mem == DFM_MEM_HOST;
  double *dr, *dq;
  OutSlot<double> oOut;
  int rc = lay_out(h, [&](Arena& a) {
    dr = hst ? a.get<double>((size_t)n * d) : nullptr;
    dq = a.get<double>(nq);
    oOut = staged(a, out, (size_t)nq * d, 1, hst);
  });
  if (rc) return rc;
  const double* r_; rc = stage_in(h, recs, dr, (size_t)n * d, mem, &r_); if (rc) return rc;
  CK(cudaMemcpyAsync(dq, q, nq * sizeof(double), cudaMemcpyHostToDevice, h->stream));      // q is always a host array
  DFM_SET_SMEM(k_percentiles, smem);
  L(k_percentiles, d, 1, 256, smem, r_, (int)n, d, dq, nq, (int)npad, oOut.at(0));
  rc = oOut.flush(h, 0, 1, mem); if (rc) return rc;
  if (!hst) CK(cudaStreamSynchronize(h->stream));                                          // (dq lives in the shared workspace)
  return finish(h, mem);
}

int dfm_percentiles_weighted(dfm_handle* h, const double* recs, const double* w, long long n, int d, const double* q, int nq, int mem,
                             double* out) {
  if (!h || !recs || !w || !q || !out || n <= 0 || d <= 0 || nq <= 0 || nq > 64 || (mem != DFM_MEM_HOST && mem != DFM_MEM_DEVICE))
    return fail(h, DFM_ERR_ARG, "dfm_percentiles_weighted: bad argument");
  for (int k = 0; k < nq; ++k)
    if (!(q[k] >= 0.0 && q[k] <= 100.0)) return fail(h, DFM_ERR_ARG, "dfm_percentiles_weighted: q outside [0, 100]");
  long long npad = 2; while (npad < n) npad <<= 1;
  const size_t smem = wpercentiles_smem_bytes(npad);
  if (smem > kMaxSmem) return fail(h, DFM_ERR_UNSUPPORTED, "dfm_percentiles_weighted: more than 16384 replications");
  CK(cudaSetDevice(h->device));
  const bool hst = mem == DFM_MEM_HOST;
  double *dr, *dw, *dq;
  OutSlot<double> oOut;
  int rc = lay_out(h, [&](Arena& a) {
    dr = hst ? a.get<double>((size_t)n * d) : nullptr;
    dw = hst ? a.get<double>((size_t)n) : nullptr;
    dq = a.get<double>(nq);
    oOut = staged(a, out, (size_t)nq * d, 1, hst);
  });
  if (rc) return rc;
  const double *r_, *w_;
  rc = stage_in(h, recs, dr, (size_t)n * d, mem, &r_); if (rc) return rc;
  rc = stage_in(h, w, dw, (size_t)n, mem, &w_); if (rc) return rc;
  CK(cudaMemcpyAsync(dq, q, nq * sizeof(double), cudaMemcpyHostToDevice, h->stream));      // q is always a host array
  DFM_SET_SMEM(k_wpercentiles, smem);
  L(k_wpercentiles, d, 1, NR_PT, smem, r_, w_, (int)n, d, dq, nq, (int)npad, oOut.at(0));
  rc = oOut.flush(h, 0, 1, mem); if (rc) return rc;
  if (!hst) CK(cudaStreamSynchronize(h->stream));                                          // (dq lives in the shared workspace)
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
