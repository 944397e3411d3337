// ctu_driver.cu -- device-resident closed-loop intra CTU search (SURVEY §8f rank 2): kernels and the C ABI of
// include/kvz_cuda_ctu.h.  The algorithm lives in csrc/ctu/*.h (single source, see ctu_common.h).
//
// Execution: one CTA works on one CTU at a time.  A picture is ONE launch of persistent CTAs that draw CTUs from a
// ticket counter in wavefront order (anti-diagonals d = x + 2y).  CTU (x, y) needs (x-1, y) and (x+1, y-1) --
// reconstructed border pixels, CU records, SAO parameters and the real coder's context models (WPP) -- and waits for
// them on the per-row progress counters (release/acquire through L2).  Tickets are handed out in dependency order and
// only to resident CTAs, so a waiting CTA always waits for CTUs that are already being worked on: no deadlock for
// any grid size.  Every picture has its own stream, so the pictures in flight (all-intra pictures are independent)
// share the GPU; after the search one launch applies SAO (final picture) and the results are copied to pinned host
// memory on the same stream.
//
// Memory per picture slot: source / reconstruction / final planes, the per-4x4 CU records, 12 KB of coefficients per
// CTU, and one work tree (CtuWork, 5 levels) per persistent CTA.
//
// The kernels are instantiated for 8-bit (uint8_t) and 10-bit (uint16_t) samples; kvz_cuda_ctu_open picks the pair
// that matches kvz_cuda_ctu_config.bitdepth, and every buffer of a slot is sized in samples of that type.
#include <time.h>
#include <condition_variable>
#include <mutex>
#include <new>
#include <vector>

#include "common.cuh"
#include "../../include/kvz_cuda_ctu.h"
#include "ctu/ctu_frame.h"

using namespace kvzctu;

static_assert(sizeof(kvz_cuda_ctu_config) == sizeof(CtuConfig), "config layout");
static_assert(sizeof(kvz_cuda_ctu_cu) == sizeof(CuRec), "cu layout");
static_assert(sizeof(kvz_cuda_ctu_sao) == sizeof(SaoRec), "sao layout");

namespace {

constexpr int kThreads = 128;
// three CTAs per SM: registers (168 x 128 threads) and shared memory (228 KB per SM, 1 KB reserved per CTA)
static_assert(sizeof(CtuST<uint8_t>) + 1024 + 64 <= 228 * 1024 / 3, "CtuST<uint8_t> no longer fits three CTAs per SM");
static_assert(sizeof(CtuST<uint16_t>) + 1024 + 64 <= 228 * 1024 / 3, "CtuST<uint16_t> no longer fits three CTAs per SM");
#if !defined(KVZ_CTU_PROF)
static_assert(sizeof(CtuST<uint8_t>) == 74960, "the 8-bit shared-memory layout changed");
#endif

template <typename Pix> struct KernelArgs {
  const CtuTables *T;
  CtuConfig cfg;
  FrameDevT<Pix> F;
  CtuWorkT<Pix> *work;      // [grid]
  SaoStats *sao_stats;     // [grid]
  uint8_t *dbg_ctx;        // [nctu][184] or NULL
  const uint16_t *order;   // [nctu][2]: CTU coordinates by ticket (wavefront order)
  int *sync;               // [0] ticket counter, [1 + cy] CTUs finished in row cy, [1 + hlcu] CTAs that have left
  int nctu;
  volatile unsigned long long *host_note;   // pinned host memory: [0] completion sequence number, [1] start, [2] end (globaltimer ns)
  unsigned long long seq;
  unsigned long long *prof;  // [PR_N + 1] phase cycles (diagnostic build only), last: CTA lifetime
  int *sm_counter;           // [256] CTAs started per SM so far: spreads the leader warps of co-resident CTAs
};

// Polling load: relaxed, from L2 (an acquire load invalidates the SM's whole L1 -- CCTL.IVALL -- on every poll, which
// also empties the L1 of the other CTAs working on that SM); the acquire fence follows once the wait is over.
__device__ __forceinline__ int ld_relaxed(const int *p)
{
  int v;
  asm volatile("ld.relaxed.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void fence_acquire() { asm volatile("fence.acq_rel.gpu;" ::: "memory"); }
__device__ __forceinline__ unsigned long long global_timer_ns()
{
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ void st_release(int *p, int v) { asm volatile("st.release.gpu.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }

__device__ __forceinline__ unsigned sm_id() { unsigned v; asm volatile("mov.u32 %0, %%smid;" : "=r"(v)); return v; }

template <typename Pix>
__global__ void __launch_bounds__(kThreads, 3) ctu_frame_kernel(const __grid_constant__ KernelArgs<Pix> a)
{
  CtuST<Pix> *S = reinterpret_cast<CtuST<Pix> *>(ctu_smem_raw);
  __shared__ int s_ticket;
  if (threadIdx.x == 0) S->leader_tid = 32 * (atomicAdd(a.sm_counter + (sm_id() & 255), 1) & 3);
  __syncthreads();
  CtxT<Pix> c = { a.T, &a.cfg, a.work + blockIdx.x, S };
#if defined(KVZ_CTU_PROF)
  const long long cta_t0 = clock64();
  if (threadIdx.x == 0) for (int i = 0; i < PR_N; ++i) S->prof[i] = 0;
#endif
  for (;;) {
    if (threadIdx.x == 0) s_ticket = atomicAdd(a.sync, 1);
    __syncthreads();
    const int t = s_ticket;
    if (t >= a.nctu) break;
    if (t == 0 && threadIdx.x == 0) a.host_note[1] = global_timer_ns();
    const int cx = a.order[2 * t], cy = a.order[2 * t + 1];
    {
      PROF_T0(PR_WAIT);
      if (threadIdx.x == 0) {
        // left neighbour: cx CTUs of this row are finished; above: the row has passed the top-right neighbour
        const int need_up = cy > 0 ? min(cx + 2, a.F.wlcu) : 0;
        while (ld_relaxed(a.sync + 1 + cy) < cx) __nanosleep(400);
        if (cy > 0) while (ld_relaxed(a.sync + cy) < need_up) __nanosleep(400);
        fence_acquire();
      }
      __syncthreads();
      PROF_ADD(S, PR_WAIT);
    }
    if (a.dbg_ctx) {
      for (int i = threadIdx.x; i < CTX_COUNT; i += blockDim.x) a.dbg_ctx[(size_t)(cy * a.F.wlcu + cx) * CTX_COUNT + i] = CTU_LD_FRAME(&a.F.row_ctx[cy].ctx[i]);
    }
    // SAO statistics in shared memory (the arena is idle after the search): block-scope atomics, no L1 staleness
    ctu_job(c, &a.F, reinterpret_cast<SaoStats *>(S->arena), cx, cy);
    __syncthreads();
    if (threadIdx.x == 0) { __threadfence(); st_release(a.sync + 1 + cy, cx + 1); }
  }
#if defined(KVZ_CTU_PROF)
  if (threadIdx.x == 0 && a.prof) {
    for (int i = 0; i < PR_N; ++i) atomicAdd(a.prof + i, (unsigned long long)S->prof[i]);
    atomicAdd(a.prof + PR_N, (unsigned long long)(clock64() - cta_t0));
  }
#endif
  // The last CTA to leave tells the host: no event follows the launch in the stream (it would sit at the head of the
  // stream's hardware queue until the launch is over and hold back the pictures of the streams behind it).
  if (threadIdx.x == 0) {
    __threadfence();
    if (atomicAdd(a.sync + 1 + a.F.hlcu, 1) == (int)gridDim.x - 1) {
      a.host_note[2] = global_timer_ns();
      __threadfence_system();
      a.host_note[0] = a.seq;
    }
  }
}

template <typename Pix>
__global__ void __launch_bounds__(kThreads) ctu_sao_apply_kernel(const __grid_constant__ KernelArgs<Pix> a)
{
  const int cy = blockIdx.x / a.F.wlcu, cx = blockIdx.x % a.F.wlcu;
  ctu_sao_apply(&a.cfg, &a.F, cx, cy);
}

struct Slot {
  int state = 0;                 // 0 free, 1 submitted
  cudaStream_t stream = nullptr;
  cudaEvent_t done = nullptr;
  volatile unsigned long long *h_note = nullptr;   // pinned: written by the search launch's last CTA
  unsigned long long seq = 0;
  bool resident = false;
  // device
  uint8_t *d_planes = nullptr;   // src | rec | out | dbg, each w*h*3/2 samples
  uint8_t *d_bufs = nullptr;     // hor / ver buffers
  CuRec *d_cu = nullptr;
  int16_t *d_coeff = nullptr;
  SaoRec *d_sao = nullptr;
  CabacState *d_row_ctx = nullptr;
  void *d_work = nullptr;        // CtuWorkT<Pix>[grid]
  SaoStats *d_stats = nullptr;
  int *d_sync = nullptr;
  uint8_t *d_dbg_ctx = nullptr;
  // pinned host
  uint8_t *h_src = nullptr;      // staging for the upload (bytes, samples of the configured type)
  uint8_t *h_out = nullptr, *h_dbg = nullptr;
  CuRec *h_cu = nullptr;
  int16_t *h_coeff = nullptr;
  SaoRec *h_sao = nullptr;
  CabacState *h_row_ctx = nullptr;
  uint8_t *h_dbg_ctx = nullptr;
  KernelArgs<uint8_t> args8;     // the arguments of the instantiation in use
  KernelArgs<uint16_t> args16;
};
template <typename Pix> KernelArgs<Pix> &args_of(Slot &s);
template <> KernelArgs<uint8_t> &args_of<uint8_t>(Slot &s) { return s.args8; }
template <> KernelArgs<uint16_t> &args_of<uint16_t>(Slot &s) { return s.args16; }

}  // namespace

struct kvz_cuda_ctu_enc {
  CtuConfig cfg;
  CtuTables *d_tables = nullptr;
  uint16_t *d_order = nullptr;
  unsigned long long *d_prof = nullptr;
  int *d_sm_counter = nullptr;
  int wl = 0, hl = 0, max_diag = 0, grid = 0;
  int pix = 1;                   // bytes per sample: 1 (8-bit) or 2 (10-bit)
  size_t plane_bytes = 0, smem = 0;
  bool debug = false;
  std::vector<Slot> slots;
  std::mutex mtx;
  std::condition_variable cv;
  std::atomic<uint64_t> launches{0};
};

#define CTU_CHECK_PTR(expr)                                                                                         \
  do {                                                                                                              \
    cudaError_t e__ = (expr);                                                                                       \
    if (e__ != cudaSuccess) {                                                                                       \
      kvzc::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__), __FILE__, __LINE__);                 \
      kvz_cuda_ctu_close(e);                                                                                        \
      return nullptr;                                                                                               \
    }                                                                                                               \
  } while (0)

extern "C" {

int kvz_cuda_ctu_config_supported(const kvz_cuda_ctu_config *c)
{
  if (!c) return -1;
  if (c->width < 8 || c->height < 8 || (c->width & 7) || (c->height & 7) || c->width > 16384 || c->height > 16384) return -1;
  if (c->rdo < 0 || c->rdo > 3) return -1;
  if (c->pu_depth_intra_min < 1 || c->pu_depth_intra_max > 4 || c->pu_depth_intra_min > c->pu_depth_intra_max) return -1;
  if (c->qp < 0 || c->qp > 51) return -1;
  if (c->bitdepth != 0 && c->bitdepth != 8 && c->bitdepth != 10) return -1;
  return 0;
}

void kvz_cuda_ctu_close(kvz_cuda_ctu_enc *e)
{
  if (!e) return;
  for (Slot &s : e->slots) {
    if (s.stream) cudaStreamSynchronize(s.stream);
    cudaFree(s.d_planes); cudaFree(s.d_bufs); cudaFree(s.d_cu); cudaFree(s.d_coeff); cudaFree(s.d_sao); cudaFree(s.d_row_ctx);
    cudaFree(s.d_work); cudaFree(s.d_stats); cudaFree(s.d_sync); cudaFree(s.d_dbg_ctx);
    cudaFreeHost(s.h_src); cudaFreeHost(s.h_out); cudaFreeHost(s.h_dbg); cudaFreeHost(s.h_cu); cudaFreeHost(s.h_coeff); cudaFreeHost(s.h_sao);
    cudaFreeHost(s.h_row_ctx); cudaFreeHost(s.h_dbg_ctx);
    if (s.done) cudaEventDestroy(s.done);
    cudaFreeHost((void *)s.h_note);
    if (s.stream) cudaStreamDestroy(s.stream);
  }
#if defined(KVZ_CTU_PROF)
  if (e->d_prof) {
    static const char *names[PR_N + 1] = { "load", "search(total)", "store", "deblock", "sao", "track", "  refs", "  satd(rough)", "  replay",
      "  quantize_residual(4x4 batches)", "  quantize_residual(8x8 batches)", "  quantize_residual(16x16 batches)",
      "  quantize_residual(32x32 batches)", "  cost(leader)", "  copies",
      "    rdo job coeff bits(leader's team)", "wait(deps)", "  chroma search(total)", "  rdo loop(total)", "  winner write-back", "CTA lifetime" };
    unsigned long long h[PR_N + 1];
    if (cudaMemcpy(h, e->d_prof, sizeof(h), cudaMemcpyDeviceToHost) == cudaSuccess) {
      fprintf(stderr, "kvz-cuda-ctu phase profile (leader-thread cycles summed over CTAs; nested phases indented):\n");
      for (int i = 0; i <= PR_N; ++i) fprintf(stderr, "  %-32s %14llu  %5.1f%%\n", names[i], h[i], 100.0 * (double)h[i] / (double)(h[PR_N] ? h[PR_N] : 1));
    }
    cudaFree(e->d_prof);
  }
#endif
  cudaFree(e->d_tables); cudaFree(e->d_order); cudaFree(e->d_sm_counter);
  delete e;
}

}  // extern "C"

// kernel arguments of a slot whose buffers are allocated: planes and border buffers in samples of Pix
template <typename Pix> static void init_args(kvz_cuda_ctu_enc *e, Slot &s, KernelArgs<Pix> &a)
{
  const int W = e->cfg.width, H = e->cfg.height;
  a.T = e->d_tables;
  a.work = (CtuWorkT<Pix> *)s.d_work; a.sao_stats = s.d_stats; a.dbg_ctx = s.d_dbg_ctx;
  a.order = e->d_order; a.sync = s.d_sync; a.nctu = e->wl * e->hl; a.prof = e->d_prof; a.sm_counter = e->d_sm_counter;
  FrameDevT<Pix> &F = a.F;
  const size_t ysz = (size_t)W * H, csz = ysz / 4, plane = ysz + 2 * csz;
  Pix *p = (Pix *)s.d_planes;
  F.src_y = p; F.src_u = p + ysz; F.src_v = p + ysz + csz; p += plane;
  F.rec_y = p; F.rec_u = p + ysz; F.rec_v = p + ysz + csz; p += plane;
  F.out_y = p; F.out_u = p + ysz; F.out_v = p + ysz + csz; p += plane;
  if (e->debug) { F.dbg_y = p; F.dbg_u = p + ysz; F.dbg_v = p + ysz + csz; } else { F.dbg_y = F.dbg_u = F.dbg_v = nullptr; }
  Pix *b = (Pix *)s.d_bufs;
  F.hor_y = b; b += (size_t)W * e->hl; F.hor_u = b; b += (size_t)(W / 2) * e->hl; F.hor_v = b; b += (size_t)(W / 2) * e->hl;
  F.ver_y = b; b += (size_t)H * e->wl; F.ver_u = b; b += (size_t)(H / 2) * e->wl; F.ver_v = b;
  F.cu = s.d_cu; F.coeff = s.d_coeff; F.sao = s.d_sao; F.row_ctx = s.d_row_ctx;
  F.cu_stride = e->wl * 16; F.wlcu = e->wl; F.hlcu = e->hl;
}

extern "C" {

kvz_cuda_ctu_enc *kvz_cuda_ctu_open(const kvz_cuda_ctu_config *cfg, int slots)
{
  if (kvz_cuda_ctu_config_supported(cfg)) { kvzc::set_error("kvz_cuda_ctu_open: configuration outside the driver's scope"); return nullptr; }
  if (kvzc::g_device < 0 && kvz_cuda_init(-1) != 0) return nullptr;
  kvz_cuda_ctu_enc *e = new (std::nothrow) kvz_cuda_ctu_enc;
  if (!e) return nullptr;
  memcpy(&e->cfg, cfg, sizeof(CtuConfig));
  const int W = cfg->width, H = cfg->height;
  e->wl = (W + 63) / 64; e->hl = (H + 63) / 64;
  // tickets: CTUs by anti-diagonal d = x + 2y, rows ascending inside a diagonal
  std::vector<uint16_t> order;
  e->max_diag = 0;
  for (int d = 0; d < e->wl + 2 * (e->hl - 1); ++d) {
    const int lo = d - (e->wl - 1) > 0 ? (d - (e->wl - 1) + 1) / 2 : 0, hi = d / 2 < e->hl - 1 ? d / 2 : e->hl - 1;
    if (hi - lo + 1 > e->max_diag) e->max_diag = hi - lo + 1;
    for (int cy = lo; cy <= hi; ++cy) { order.push_back((uint16_t)(d - 2 * cy)); order.push_back((uint16_t)cy); }
  }
  // persistent CTAs per picture: 40 % of the widest diagonal (the average wavefront is about half of it; a smaller grid
  // leaves fewer CTAs waiting idle and lets more pictures be resident at once)
  e->grid = (e->max_diag * 2 + 4) / 5;
  if (e->grid < 1) e->grid = 1;
  e->pix = cfg->bitdepth == 10 ? 2 : 1;
  e->plane_bytes = (size_t)W * H * 3 / 2 * e->pix;
  e->smem = e->pix == 2 ? sizeof(CtuST<uint16_t>) : sizeof(CtuST<uint8_t>);
  e->debug = getenv("KVZ_CUDA_CTU_DEBUG") != nullptr;
  {
    CtuTables *ht = new CtuTables;
    ctu_tables_init(ht);
    cudaError_t err = cudaMalloc(&e->d_tables, sizeof(CtuTables));
    if (err == cudaSuccess) err = cudaMemcpy(e->d_tables, ht, sizeof(CtuTables), cudaMemcpyHostToDevice);
    delete ht;
    CTU_CHECK_PTR(err);
  }
#if defined(KVZ_CTU_PROF)
  CTU_CHECK_PTR(cudaMalloc(&e->d_prof, (PR_N + 1) * sizeof(unsigned long long)));
  CTU_CHECK_PTR(cudaMemset(e->d_prof, 0, (PR_N + 1) * sizeof(unsigned long long)));
#endif
  CTU_CHECK_PTR(cudaMalloc(&e->d_sm_counter, 256 * sizeof(int)));
  CTU_CHECK_PTR(cudaMemset(e->d_sm_counter, 0, 256 * sizeof(int)));
  CTU_CHECK_PTR(cudaMalloc(&e->d_order, order.size() * sizeof(uint16_t)));
  CTU_CHECK_PTR(cudaMemcpy(e->d_order, order.data(), order.size() * sizeof(uint16_t), cudaMemcpyHostToDevice));
  if (e->pix == 2) CTU_CHECK_PTR(cudaFuncSetAttribute(ctu_frame_kernel<uint16_t>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)e->smem));
  else CTU_CHECK_PTR(cudaFuncSetAttribute(ctu_frame_kernel<uint8_t>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)e->smem));
  e->slots.resize(slots > 0 ? (slots > 512 ? 512 : slots) : 1);
  const size_t nctu = (size_t)e->wl * e->hl;
  const size_t cu_n = (size_t)(e->wl * 16) * (e->hl * 16);
  const size_t buf_bytes = (((size_t)W * e->hl + (size_t)H * e->wl) * 2 + 64) * e->pix;    // Y + U + V rows (columns): w + w/2 + w/2
  for (Slot &s : e->slots) {
    CTU_CHECK_PTR(cudaStreamCreateWithFlags(&s.stream, cudaStreamNonBlocking));
    CTU_CHECK_PTR(cudaEventCreateWithFlags(&s.done, cudaEventDisableTiming));
    CTU_CHECK_PTR(cudaHostAlloc((void **)&s.h_note, 64, cudaHostAllocDefault));
    memset((void *)s.h_note, 0, 64);
    CTU_CHECK_PTR(cudaMalloc(&s.d_planes, e->plane_bytes * 4));
    CTU_CHECK_PTR(cudaMalloc(&s.d_bufs, buf_bytes));
    CTU_CHECK_PTR(cudaMalloc(&s.d_cu, cu_n * sizeof(CuRec)));
    CTU_CHECK_PTR(cudaMalloc(&s.d_coeff, nctu * 6144 * sizeof(int16_t)));
    CTU_CHECK_PTR(cudaMalloc(&s.d_sao, nctu * 2 * sizeof(SaoRec)));
    CTU_CHECK_PTR(cudaMalloc(&s.d_row_ctx, e->hl * sizeof(CabacState)));
    CTU_CHECK_PTR(cudaMalloc(&s.d_work, (size_t)e->grid * (e->pix == 2 ? sizeof(CtuWorkT<uint16_t>) : sizeof(CtuWorkT<uint8_t>))));
    CTU_CHECK_PTR(cudaMalloc(&s.d_stats, (size_t)e->grid * sizeof(SaoStats)));
    CTU_CHECK_PTR(cudaMalloc(&s.d_sync, (size_t)(e->hl + 2) * sizeof(int)));
    CTU_CHECK_PTR(cudaMemset(s.d_sao, 0, nctu * 2 * sizeof(SaoRec)));
    CTU_CHECK_PTR(cudaMemset(s.d_planes, 0, e->plane_bytes * 4));
    CTU_CHECK_PTR(cudaMemset(s.d_bufs, 0, buf_bytes));
    CTU_CHECK_PTR(cudaHostAlloc(&s.h_src, e->plane_bytes, cudaHostAllocDefault));
    CTU_CHECK_PTR(cudaHostAlloc(&s.h_out, e->plane_bytes, cudaHostAllocDefault));
    CTU_CHECK_PTR(cudaHostAlloc(&s.h_cu, cu_n * sizeof(CuRec), cudaHostAllocDefault));
    CTU_CHECK_PTR(cudaHostAlloc(&s.h_coeff, nctu * 6144 * sizeof(int16_t), cudaHostAllocDefault));
    CTU_CHECK_PTR(cudaHostAlloc(&s.h_sao, nctu * 2 * sizeof(SaoRec), cudaHostAllocDefault));
    CTU_CHECK_PTR(cudaHostAlloc(&s.h_row_ctx, e->hl * sizeof(CabacState), cudaHostAllocDefault));
    if (e->debug) {
      CTU_CHECK_PTR(cudaMalloc(&s.d_dbg_ctx, nctu * CTX_COUNT));
      CTU_CHECK_PTR(cudaHostAlloc(&s.h_dbg_ctx, nctu * CTX_COUNT, cudaHostAllocDefault));
      CTU_CHECK_PTR(cudaHostAlloc(&s.h_dbg, e->plane_bytes, cudaHostAllocDefault));
    }
    if (e->pix == 2) init_args(e, s, s.args16); else init_args(e, s, s.args8);
  }
  return e;
}

}  // extern "C"

// the search launch of a submitted picture
template <typename Pix> static int launch_search(kvz_cuda_ctu_enc *e, Slot &s, double lambda, double lambda_sqrt, int qp)
{
  KernelArgs<Pix> &a = args_of<Pix>(s);
  a.cfg = e->cfg;
  a.cfg.lambda = lambda; a.cfg.lambda_sqrt = lambda_sqrt; a.cfg.qp = qp;
  a.host_note = s.h_note;
  a.seq = s.seq;
  ctu_frame_kernel<Pix><<<e->grid, kThreads, e->smem, s.stream>>>(a);
  e->launches.fetch_add(1, std::memory_order_relaxed);
  kvzc::g_launches.fetch_add(1, std::memory_order_relaxed);
  return 0;
}

extern "C" {

// common part of the two submit calls: `resident`: the planes are device memory and the results stay on the device.
// Samples are uint8_t or uint16_t (cfg.bitdepth), strides in samples.
static int submit_picture(kvz_cuda_ctu_enc *e, const void *y, const void *u, const void *v, int stride_y, int stride_c,
                          const uint8_t *ctx_init, double lambda, double lambda_sqrt, int qp, bool resident)
{
  KVZC_ARG(e && y && u && v && ctx_init && stride_y >= e->cfg.width && stride_c >= e->cfg.width / 2);
  int id = -1;
  {
    std::unique_lock<std::mutex> lock(e->mtx);
    e->cv.wait(lock, [&] { for (size_t i = 0; i < e->slots.size(); ++i) if (e->slots[i].state == 0) { id = (int)i; return true; } return false; });
    e->slots[id].state = 1;
  }
  Slot &s = e->slots[id];
  const int W = e->cfg.width, H = e->cfg.height;
  const size_t px = (size_t)e->pix;
  const size_t ysz = (size_t)W * H * px, csz = ysz / 4;           // bytes
  const size_t wb = (size_t)W * px, sy = (size_t)stride_y * px, sc = (size_t)stride_c * px;
  const uint8_t *yb = (const uint8_t *)y, *ub = (const uint8_t *)u, *vb = (const uint8_t *)v;
  cudaStream_t st = s.stream;
  uint8_t *d_src = s.d_planes;        // (the source planes come first)
  if (resident) {
    KVZC_CHECK(cudaMemcpy2DAsync(d_src, wb, yb, sy, wb, H, cudaMemcpyDeviceToDevice, st));
    KVZC_CHECK(cudaMemcpy2DAsync(d_src + ysz, wb / 2, ub, sc, wb / 2, H / 2, cudaMemcpyDeviceToDevice, st));
    KVZC_CHECK(cudaMemcpy2DAsync(d_src + ysz + csz, wb / 2, vb, sc, wb / 2, H / 2, cudaMemcpyDeviceToDevice, st));
  } else {
    for (int r = 0; r < H; ++r) memcpy(s.h_src + (size_t)r * wb, yb + (size_t)r * sy, wb);
    for (int r = 0; r < H / 2; ++r) {
      memcpy(s.h_src + ysz + (size_t)r * (wb / 2), ub + (size_t)r * sc, wb / 2);
      memcpy(s.h_src + ysz + csz + (size_t)r * (wb / 2), vb + (size_t)r * sc, wb / 2);
    }
    KVZC_CHECK(cudaMemcpyAsync(d_src, s.h_src, e->plane_bytes, cudaMemcpyHostToDevice, st));
  }
  for (int r = 0; r < e->hl; ++r) { memcpy(s.h_row_ctx[r].ctx, ctx_init, CTX_COUNT); s.h_row_ctx[r].update = 0; memset(s.h_row_ctx[r].pad, 0, sizeof(s.h_row_ctx[r].pad)); }
  KVZC_CHECK(cudaMemcpyAsync(s.d_row_ctx, s.h_row_ctx, e->hl * sizeof(CabacState), cudaMemcpyHostToDevice, st));
  KVZC_CHECK(cudaMemsetAsync(s.d_cu, 0, (size_t)(e->wl * 16) * (e->hl * 16) * sizeof(CuRec), st));
  KVZC_CHECK(cudaMemsetAsync(s.d_sync, 0, (size_t)(e->hl + 2) * sizeof(int), st));
  s.seq += 1;
  if (e->pix == 2) launch_search<uint16_t>(e, s, lambda, lambda_sqrt, qp);
  else launch_search<uint8_t>(e, s, lambda, lambda_sqrt, qp);
  KVZC_CHECK(cudaGetLastError());
  s.resident = resident;
  return id;
}

// Second half of a picture, enqueued by the waiting thread once the search launch has finished: SAO over the whole
// picture and the copies to pinned memory.  Deliberately NOT enqueued at submit time: work that depends on the (long)
// search launch would sit at the head of its hardware queue (CUDA_DEVICE_MAX_CONNECTIONS of them, 8 by default) and
// block the pictures of other streams queued behind it -- only one picture per queue would run.
static int finish_picture(kvz_cuda_ctu_enc *e, Slot &s)
{
  // sleep-poll the completion note (the host threads are needed by the encoder's CABAC stage)
  unsigned spins = 0;
  while (__atomic_load_n((const unsigned long long *)s.h_note, __ATOMIC_ACQUIRE) != s.seq) {
    if (++spins > 20) { struct timespec ts = { 0, 200000 }; nanosleep(&ts, nullptr); }
    if ((spins & 1023) == 0) { const cudaError_t err = cudaStreamQuery(s.stream); if (err != cudaSuccess && err != cudaErrorNotReady) KVZC_CHECK(err); }
  }
  cudaStream_t st = s.stream;
  if (e->pix == 2) ctu_sao_apply_kernel<uint16_t><<<e->wl * e->hl, kThreads, 0, st>>>(s.args16);
  else ctu_sao_apply_kernel<uint8_t><<<e->wl * e->hl, kThreads, 0, st>>>(s.args8);
  e->launches.fetch_add(1, std::memory_order_relaxed);
  kvzc::g_launches.fetch_add(1, std::memory_order_relaxed);
  KVZC_CHECK(cudaGetLastError());
  if (!s.resident) {
    const size_t nctu = (size_t)e->wl * e->hl;
    KVZC_CHECK(cudaMemcpyAsync(s.h_cu, s.d_cu, (size_t)(e->wl * 16) * (e->hl * 16) * sizeof(CuRec), cudaMemcpyDeviceToHost, st));
    KVZC_CHECK(cudaMemcpyAsync(s.h_coeff, s.d_coeff, nctu * 6144 * sizeof(int16_t), cudaMemcpyDeviceToHost, st));
    KVZC_CHECK(cudaMemcpyAsync(s.h_sao, s.d_sao, nctu * 2 * sizeof(SaoRec), cudaMemcpyDeviceToHost, st));
    KVZC_CHECK(cudaMemcpyAsync(s.h_out, s.d_planes + 2 * e->plane_bytes, e->plane_bytes, cudaMemcpyDeviceToHost, st));
    if (e->debug) {
      KVZC_CHECK(cudaMemcpyAsync(s.h_dbg_ctx, s.d_dbg_ctx, nctu * CTX_COUNT, cudaMemcpyDeviceToHost, st));
      KVZC_CHECK(cudaMemcpyAsync(s.h_dbg, s.d_planes + 3 * e->plane_bytes, e->plane_bytes, cudaMemcpyDeviceToHost, st));
    }
  }
  KVZC_CHECK(cudaEventRecord(s.done, st));
  KVZC_CHECK(cudaEventSynchronize(s.done));
  return 0;
}

int kvz_cuda_ctu_submit(kvz_cuda_ctu_enc *e, const uint8_t *y, const uint8_t *u, const uint8_t *v, int stride_y, int stride_c,
                        const uint8_t *ctx_init, double lambda, double lambda_sqrt, int qp)
{
  return submit_picture(e, y, u, v, stride_y, stride_c, ctx_init, lambda, lambda_sqrt, qp, false);
}

int kvz_cuda_ctu_submit_device(kvz_cuda_ctu_enc *e, const uint8_t *d_y, const uint8_t *d_u, const uint8_t *d_v, int stride_y, int stride_c,
                               const uint8_t *ctx_init, double lambda, double lambda_sqrt, int qp)
{
  return submit_picture(e, d_y, d_u, d_v, stride_y, stride_c, ctx_init, lambda, lambda_sqrt, qp, true);
}

int kvz_cuda_ctu_wait_device(kvz_cuda_ctu_enc *e, int slot, kvz_cuda_ctu_device_result *out)
{
  KVZC_ARG(e && out && slot >= 0 && slot < (int)e->slots.size() && e->slots[slot].state == 1);
  Slot &s = e->slots[slot];
  if (int rc = finish_picture(e, s)) return rc;
  memset(out, 0, sizeof(*out));
  out->cu = (const kvz_cuda_ctu_cu *)s.d_cu;
  out->coeff = s.d_coeff;
  out->sao = (const kvz_cuda_ctu_sao *)s.d_sao;
  out->rec = s.d_planes + 2 * e->plane_bytes;
  out->cu_stride = e->wl * 16;
  out->width_in_lcu = e->wl; out->height_in_lcu = e->hl;
  out->search_kernel_ms = (float)((double)(s.h_note[2] - s.h_note[1]) * 1e-6);   // globaltimer ns of first / last CTA
  return 0;
}

int kvz_cuda_ctu_wait(kvz_cuda_ctu_enc *e, int slot, kvz_cuda_ctu_result *out)
{
  KVZC_ARG(e && out && slot >= 0 && slot < (int)e->slots.size() && e->slots[slot].state == 1);
  Slot &s = e->slots[slot];
  if (int rc = finish_picture(e, s)) return rc;
  const size_t ysz = (size_t)e->cfg.width * e->cfg.height * e->pix, csz = ysz / 4;     // bytes
  memset(out, 0, sizeof(*out));
  out->cu = (const kvz_cuda_ctu_cu *)s.h_cu;
  out->cu_stride = e->wl * 16;
  out->width_in_lcu = e->wl; out->height_in_lcu = e->hl;
  out->coeff = s.h_coeff;
  out->sao = (const kvz_cuda_ctu_sao *)s.h_sao;
  out->rec_y = s.h_out; out->rec_u = s.h_out + ysz; out->rec_v = s.h_out + ysz + csz;
  if (e->debug) { out->dbg_ctx = s.h_dbg_ctx; out->dbg_y = s.h_dbg; out->dbg_u = s.h_dbg + ysz; out->dbg_v = s.h_dbg + ysz + csz; }
  return 0;
}

void kvz_cuda_ctu_release(kvz_cuda_ctu_enc *e, int slot)
{
  if (!e || slot < 0 || slot >= (int)e->slots.size()) return;
  {
    std::lock_guard<std::mutex> lock(e->mtx);
    e->slots[slot].state = 0;
  }
  e->cv.notify_one();
}

uint64_t kvz_cuda_ctu_launches(const kvz_cuda_ctu_enc *e) { return e ? e->launches.load() : 0; }

}  // extern "C"
