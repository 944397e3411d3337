// ctu_frame_probe.cu -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
//
// Runs the back half of the CTU search driver's CTU job (ctu_job of kvazaar_b200/csrc/ctu/ctu_frame.h with search_ctu
// replaced by INJECTED decisions: ctu_store, ctu_deblock, ctu_sao_search, ctu_track_models) over a whole picture, then
// ctu_sao_apply over every CTU, and returns every output, so that tests/test_ctu_frame_stage.py can compare them CTU by
// CTU with the reference's own CTU job on the same decisions.  One source, two builds (make probe):
//   * nvcc, sm_90a (tests/cuda/libkvzctu_frame_probe.so): one 128-thread CTA per CTU with the driver's launch bounds and
//     shared-memory state, one launch per wavefront anti-diagonal d = x + 2y -- exactly the CTUs the driver may run at
//     the same time; the CTUs each of them depends on, (x - 1, y) and (x + 1, y - 1), finished in an earlier launch;
//   * g++ -x c++ (tests/hostsim/libkvzctu_frame_probe_host.so): the one-thread CTA, the same diagonals in turn (or the
//     CTUs in raster order).
// It lives outside kvazaar_b200/csrc so that the product library never contains it.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include <vector>

#include "../../kvazaar_b200/csrc/ctu/ctu_frame.h"

using namespace kvzctu;

namespace {

struct FrameProbeArgs {
  const CtuTables *T;
  const CtuConfig *cfg;
  const CuRec *cu;              // [height / 4][width / 4]: the injected records
  const void *rec;              // pre-deblock reconstruction, Y, U, V planes back to back, stride = width (/2)
  const int16_t *coeff;         // per CTU (raster): y[4096] u[1024] v[1024], lcu_coeff_t layout
  const int32_t *leader;        // per CTU: leader_tid
  uint8_t *ctx_start, *ctx_end; // per CTU: CTX_COUNT model bytes
  int fill;
};

// ctu_job with the search replaced by injection; `W` is the CTA's work area
template <typename Pix> CTU_FN_NOINLINE void probe_ctu(const FrameProbeArgs &a, const FrameDevT<Pix> *F, CtuST<Pix> *S, CtuWorkT<Pix> *W, int cx, int cy)
{
  const int ctu = cy * F->wlcu + cx;
  // the shared state (arena included) and the work area hold a known byte: a stage that reads what it did not write sees it
  #pragma unroll 1
  for (int i = CTU_TID; i < (int)sizeof(CtuST<Pix>); i += CTU_NT) ((uint8_t *)S)[i] = (uint8_t)a.fill;
  #pragma unroll 1
  for (int i = CTU_TID; i < (int)sizeof(CtuWorkT<Pix>); i += CTU_NT) ((uint8_t *)W)[i] = (uint8_t)a.fill;
  CTU_SYNC();
  if (CTU_TID == 0) S->leader_tid = a.leader[ctu];
  CTU_SYNC();
  // 1. the configuration (ctu_job)
  #pragma unroll 1
  for (int i = CTU_TID; i < (int)(sizeof(CtuConfig) / 4); i += CTU_NT) ((uint32_t *)&S->cfg)[i] = ((const uint32_t *)a.cfg)[i];
  CTU_LEADER S->W = W;
  CTU_SYNC();
  #pragma unroll 1
  for (int i = CTU_TID; i < CTX_COUNT; i += CTU_NT) a.ctx_start[(size_t)ctu * CTX_COUNT + i] = CTU_LD_FRAME(&F->row_ctx[cy].ctx[i]);
  // 2. ctu_load
  ctu_load(S, F, cx, cy);
  sm_tables_load(&S->tb, a.T);
  // 3. the decisions, where search_ctu leaves them: level 0 of the work tree
  {
    LcuLevel<Pix> *L0 = &S->lv[0];
    const int Wd = a.cfg->width, H = a.cfg->height, x = cx * 64, y = cy * 64;
    const int x_max = imin(x + 64, Wd) - x, y_max = imin(y + 64, H) - y;
    const Pix *ry = (const Pix *)a.rec, *ru = ry + (size_t)Wd * H, *rv = ru + (size_t)(Wd / 2) * (H / 2);
    #pragma unroll 1
    for (int e = CTU_TID; e < 256; e += CTU_NT) {
      const int sx = e & 15, sy = e >> 4;
      if (4 * sx < x_max && 4 * sy < y_max) *cu_at(L0, 4 * sx, 4 * sy) = a.cu[((y >> 2) + sy) * (Wd >> 2) + (x >> 2) + sx];
    }
    #pragma unroll 1
    for (int e = CTU_TID; e < 64 * 64; e += CTU_NT) {
      const int yy = e >> 6, xx = e & 63;
      if (xx < x_max && yy < y_max) L0->rec_y[e] = ry[(size_t)(y + yy) * Wd + x + xx];
      L0->coeff_y[e] = a.coeff[(size_t)ctu * 6144 + e];
    }
    #pragma unroll 1
    for (int e = CTU_TID; e < 32 * 32; e += CTU_NT) {
      const int yy = e >> 5, xx = e & 31;
      if (xx < x_max / 2 && yy < y_max / 2) {
        L0->rec_u[e] = ru[(size_t)(y / 2 + yy) * (Wd / 2) + x / 2 + xx];
        L0->rec_v[e] = rv[(size_t)(y / 2 + yy) * (Wd / 2) + x / 2 + xx];
      }
      L0->coeff_u[e] = a.coeff[(size_t)ctu * 6144 + 4096 + e];
      L0->coeff_v[e] = a.coeff[(size_t)ctu * 6144 + 5120 + e];
    }
    CTU_SYNC();
  }
  // 4. as ctu_job: store, deblocking, the SAO search with its statistics in the arena
  ctu_store(S, F, cx, cy);
#if defined(__CUDA_ARCH__)
  __threadfence();
#endif
  CTU_SYNC();
  if (S->cfg.deblock_enable) ctu_deblock(S, F, cx, cy);
  if (S->cfg.sao_type) ctu_sao_search(S, F, reinterpret_cast<SaoStats *>(S->arena), cx, cy);
  // 5. the real coder's models
  ctu_track_models(S, F, cx, cy);
  #pragma unroll 1
  for (int i = CTU_TID; i < CTX_COUNT; i += CTU_NT) a.ctx_end[(size_t)ctu * CTX_COUNT + i] = S->tmp.ctx[i];
  CTU_SYNC();
}

// the CTUs of anti-diagonal d = x + 2y, by increasing y (host and device: the launches are sized with them)
#if defined(__CUDACC__)
#define PROBE_HD __host__ __device__ inline
#else
#define PROBE_HD static inline
#endif
PROBE_HD int diag_first_y(int d, int wl) { const int lo = d - (wl - 1); return lo > 0 ? (lo + 1) / 2 : 0; }
PROBE_HD int diag_count(int d, int wl, int hl)
{
  const int y0 = diag_first_y(d, wl), y1 = hl - 1 < d / 2 ? hl - 1 : d / 2;
  return y1 >= y0 ? y1 - y0 + 1 : 0;
}

// the frame buffers of the driver (kvz_cuda_ctu_open's per-slot layout), sized for one picture
template <typename Pix> struct FrameBufs {
  size_t ny, nc, ncu, nctu;
  int wl, hl, cu_stride;
  void init(int w, int h)
  {
    wl = (w + 63) / 64; hl = (h + 63) / 64; cu_stride = wl * 16;
    ny = (size_t)w * h; nc = ny / 4; ncu = (size_t)cu_stride * hl * 16; nctu = (size_t)wl * hl;
  }
};

#if defined(__CUDACC__)
template <typename Pix> __global__ void __launch_bounds__(128, 3) probe_diag_kernel(const __grid_constant__ FrameProbeArgs a, const __grid_constant__ FrameDevT<Pix> F, CtuWorkT<Pix> *work, int d)
{
  const int cy = diag_first_y(d, F.wlcu) + blockIdx.x, cx = d - 2 * cy;
  probe_ctu<Pix>(a, &F, reinterpret_cast<CtuST<Pix> *>(ctu_smem_raw), work + blockIdx.x, cx, cy);
}
template <typename Pix> __global__ void __launch_bounds__(128) probe_sao_apply_kernel(const __grid_constant__ CtuConfig cfg, const __grid_constant__ FrameDevT<Pix> F)
{
  ctu_sao_apply(&cfg, &F, blockIdx.x % F.wlcu, blockIdx.x / F.wlcu);
}

#define PROBE_CHECK(expr) do { const cudaError_t e_ = (expr); if (e_ != cudaSuccess) { fprintf(stderr, "ctu_frame_probe: %s: %s\n", #expr, cudaGetErrorString(e_)); rc = -1; goto out; } } while (0)

template <typename Pix> int run(const CtuConfig *cfg, const uint8_t *ctx_init, const Pix *src, FrameProbeArgs h, int, Pix *dbk, Pix *out, SaoRec *sao, int32_t *info)
{
  int rc = 0, widest = 0;
  FrameBufs<Pix> b;
  b.init(cfg->width, cfg->height);
  std::vector<void *> bufs;
  bool ok = true;
  auto up = [&](const void *p, size_t bytes) -> void * {
    void *d = NULL;
    if (cudaMalloc(&d, bytes) != cudaSuccess) { ok = false; return NULL; }
    bufs.push_back(d);
    if (p ? cudaMemcpy(d, p, bytes, cudaMemcpyHostToDevice) != cudaSuccess : cudaMemset(d, 0, bytes) != cudaSuccess) ok = false;
    return d;
  };
  const int ndiag = (b.wl - 1) + 2 * (b.hl - 1) + 1;
  for (int d = 0; d < ndiag; ++d) widest = std::max(widest, diag_count(d, b.wl, b.hl));
  CtuTables tables;
  ctu_tables_init(&tables);
  std::vector<CabacState> rows(b.hl);
  for (auto &r : rows) { memset(&r, 0, sizeof(r)); memcpy(r.ctx, ctx_init, CTX_COUNT); }
  const size_t planes = (b.ny + 2 * b.nc) * sizeof(Pix);
  FrameProbeArgs a = h;
  FrameDevT<Pix> F;
  memset(&F, 0, sizeof(F));
  Pix *src_d, *rec_d, *out_d, *hor_d, *ver_d;
  CtuWorkT<Pix> *work = NULL;
  a.T = (const CtuTables *)up(&tables, sizeof(tables));
  a.cfg = (const CtuConfig *)up(cfg, sizeof(CtuConfig));
  a.cu = (const CuRec *)up(h.cu, (b.ny / 16) * sizeof(CuRec));
  a.rec = up(h.rec, planes);
  a.coeff = (const int16_t *)up(h.coeff, b.nctu * 6144 * sizeof(int16_t));
  a.leader = (const int32_t *)up(h.leader, b.nctu * sizeof(int32_t));
  a.ctx_start = (uint8_t *)up(NULL, b.nctu * CTX_COUNT);
  a.ctx_end = (uint8_t *)up(NULL, b.nctu * CTX_COUNT);
  src_d = (Pix *)up(src, planes);
  rec_d = (Pix *)up(NULL, planes);
  out_d = (Pix *)up(NULL, planes);
  hor_d = (Pix *)up(NULL, (size_t)b.hl * cfg->width * 2 * sizeof(Pix));
  ver_d = (Pix *)up(NULL, (size_t)b.wl * cfg->height * 2 * sizeof(Pix));
  F.cu = (CuRec *)up(NULL, b.ncu * sizeof(CuRec));
  F.coeff = (int16_t *)up(NULL, b.nctu * 6144 * sizeof(int16_t));
  F.sao = (SaoRec *)up(NULL, b.nctu * 2 * sizeof(SaoRec));
  F.row_ctx = (CabacState *)up(rows.data(), b.hl * sizeof(CabacState));
  work = (CtuWorkT<Pix> *)up(NULL, (size_t)widest * sizeof(CtuWorkT<Pix>));
  if (!ok) { fprintf(stderr, "ctu_frame_probe: device allocation or upload failed\n"); rc = -1; goto out; }
  F.src_y = src_d; F.src_u = src_d + b.ny; F.src_v = src_d + b.ny + b.nc;
  F.rec_y = rec_d; F.rec_u = rec_d + b.ny; F.rec_v = rec_d + b.ny + b.nc;
  F.out_y = out_d; F.out_u = out_d + b.ny; F.out_v = out_d + b.ny + b.nc;
  F.hor_y = hor_d; F.hor_u = hor_d + (size_t)b.hl * cfg->width; F.hor_v = F.hor_u + (size_t)b.hl * cfg->width / 2;
  F.ver_y = ver_d; F.ver_u = ver_d + (size_t)b.wl * cfg->height; F.ver_v = F.ver_u + (size_t)b.wl * cfg->height / 2;
  F.cu_stride = b.cu_stride; F.wlcu = b.wl; F.hlcu = b.hl;
  PROBE_CHECK(cudaFuncSetAttribute(probe_diag_kernel<Pix>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(CtuST<Pix>)));
  for (int d = 0; d < ndiag; ++d) {
    const int n = diag_count(d, b.wl, b.hl);
    if (!n) continue;
    probe_diag_kernel<Pix><<<n, 128, sizeof(CtuST<Pix>)>>>(a, F, work, d);
    PROBE_CHECK(cudaGetLastError());
  }
  probe_sao_apply_kernel<Pix><<<(int)b.nctu, 128>>>(*cfg, F);
  PROBE_CHECK(cudaGetLastError());
  PROBE_CHECK(cudaDeviceSynchronize());
  PROBE_CHECK(cudaMemcpy(dbk, rec_d, planes, cudaMemcpyDeviceToHost));
  PROBE_CHECK(cudaMemcpy(out, out_d, planes, cudaMemcpyDeviceToHost));
  PROBE_CHECK(cudaMemcpy(sao, F.sao, b.nctu * 2 * sizeof(SaoRec), cudaMemcpyDeviceToHost));
  PROBE_CHECK(cudaMemcpy(h.ctx_start, a.ctx_start, b.nctu * CTX_COUNT, cudaMemcpyDeviceToHost));
  PROBE_CHECK(cudaMemcpy(h.ctx_end, a.ctx_end, b.nctu * CTX_COUNT, cudaMemcpyDeviceToHost));
  info[0] = widest;
out:
  for (void *p : bufs) cudaFree(p);
  return rc;
}
#else
template <typename Pix> int run(const CtuConfig *cfg, const uint8_t *ctx_init, const Pix *src, FrameProbeArgs a, int raster, Pix *dbk, Pix *out, SaoRec *sao, int32_t *info)
{
  FrameBufs<Pix> b;
  b.init(cfg->width, cfg->height);
  CtuTables *tables = new CtuTables;
  ctu_tables_init(tables);
  a.T = tables;
  std::vector<Pix> rec(b.ny + 2 * b.nc), hor((size_t)b.hl * cfg->width * 2), ver((size_t)b.wl * cfg->height * 2);
  std::vector<CuRec> cu(b.ncu);
  std::vector<int16_t> coeff(b.nctu * 6144);
  std::vector<CabacState> rows(b.hl);
  for (auto &r : rows) { memset(&r, 0, sizeof(r)); memcpy(r.ctx, ctx_init, CTX_COUNT); }
  memset(cu.data(), 0, cu.size() * sizeof(CuRec));
  memset(sao, 0, b.nctu * 2 * sizeof(SaoRec));
  FrameDevT<Pix> F;
  memset(&F, 0, sizeof(F));
  F.src_y = src; F.src_u = src + b.ny; F.src_v = src + b.ny + b.nc;
  F.rec_y = rec.data(); F.rec_u = F.rec_y + b.ny; F.rec_v = F.rec_u + b.nc;
  F.out_y = out; F.out_u = out + b.ny; F.out_v = out + b.ny + b.nc;
  F.hor_y = hor.data(); F.hor_u = F.hor_y + (size_t)b.hl * cfg->width; F.hor_v = F.hor_u + (size_t)b.hl * cfg->width / 2;
  F.ver_y = ver.data(); F.ver_u = F.ver_y + (size_t)b.wl * cfg->height; F.ver_v = F.ver_u + (size_t)b.wl * cfg->height / 2;
  F.cu = cu.data(); F.coeff = coeff.data(); F.sao = sao; F.row_ctx = rows.data();
  F.cu_stride = b.cu_stride; F.wlcu = b.wl; F.hlcu = b.hl;
  CtuST<Pix> *S = (CtuST<Pix> *)malloc(sizeof(CtuST<Pix>));
  CtuWorkT<Pix> *W = (CtuWorkT<Pix> *)malloc(sizeof(CtuWorkT<Pix>));
  int widest = 0;
  if (raster) {
    for (int cy = 0; cy < b.hl; ++cy)
      for (int cx = 0; cx < b.wl; ++cx) probe_ctu<Pix>(a, &F, S, W, cx, cy);
  } else {
    const int ndiag = (b.wl - 1) + 2 * (b.hl - 1) + 1;
    for (int d = 0; d < ndiag; ++d) {
      const int n = diag_count(d, b.wl, b.hl), y0 = diag_first_y(d, b.wl);
      widest = std::max(widest, n);
      for (int k = 0; k < n; ++k) probe_ctu<Pix>(a, &F, S, W, d - 2 * (y0 + k), y0 + k);
    }
  }
  for (int cy = 0; cy < b.hl; ++cy)
    for (int cx = 0; cx < b.wl; ++cx) ctu_sao_apply(cfg, &F, cx, cy);
  memcpy(dbk, rec.data(), rec.size() * sizeof(Pix));
  info[0] = widest;
  free(W);
  free(S);
  delete tables;
  return 0;
}
#endif

}  // namespace

extern "C" {

// One picture: the back half of every CTU's job on the injected decisions `cu` / `rec` / `coeff` (see FrameProbeArgs for
// the layouts), the diagonals in turn (raster = 1: the CTUs in raster order, host build only), then SAO application.
// Every row's models start as ctx_init (CTX_COUNT bytes).  Samples are uint8_t at bitdepth 8 and uint16_t at bitdepth
// 10; `src` and the outputs `dbk` (the picture after deblocking) and `out` (the final picture) are Y, U, V planes back to
// back.  Per CTU: sao[2] (luma, chroma), the models at its start (ctx_start) and after its syntax (ctx_end).  info[0]:
// the most CTUs one diagonal ran at the same time (0 in raster order).  Returns 0, or -1 on a bad argument or a CUDA
// error.
int kvz_ctu_frame_probe_run(int bitdepth, const void *cfg_in, const uint8_t *ctx_init, const void *src, const void *cu, const void *rec,
                            const int16_t *coeff, const int32_t *leader, int fill, int raster, void *dbk, void *out, void *sao,
                            uint8_t *ctx_start, uint8_t *ctx_end, int32_t *info)
{
  const CtuConfig *cfg = (const CtuConfig *)cfg_in;
  if (!cfg || !ctx_init || !src || !cu || !rec || !coeff || !leader || !dbk || !out || !sao || !ctx_start || !ctx_end || !info) return -1;
  if (bitdepth != 8 && bitdepth != 10) return -1;
  if (cfg->bitdepth != bitdepth && !(bitdepth == 8 && cfg->bitdepth == 0)) return -1;
  if (!cfg->wpp || cfg->width <= 0 || cfg->height <= 0 || (cfg->width & 7) || (cfg->height & 7)) return -1;
  if (cfg->qp < 0 || cfg->qp > 51 || cfg->sao_type < 0 || cfg->sao_type > 3) return -1;
  if (cfg->deblock_beta < -6 || cfg->deblock_beta > 6 || cfg->deblock_tc < -6 || cfg->deblock_tc > 6) return -1;
#if defined(__CUDACC__)
  if (raster) return -1;
#endif
  const int nctu = ((cfg->width + 63) / 64) * ((cfg->height + 63) / 64);
  for (int i = 0; i < nctu; ++i) if (leader[i] < 0 || leader[i] > 96 || (leader[i] & 31)) return -1;
  FrameProbeArgs a = { NULL, cfg, (const CuRec *)cu, rec, coeff, leader, ctx_start, ctx_end, fill };
  if (bitdepth == 8) return run<uint8_t>(cfg, ctx_init, (const uint8_t *)src, a, raster, (uint8_t *)dbk, (uint8_t *)out, (SaoRec *)sao, info);
  return run<uint16_t>(cfg, ctx_init, (const uint16_t *)src, a, raster, (uint16_t *)dbk, (uint16_t *)out, (SaoRec *)sao, info);
}

}  // extern "C"
