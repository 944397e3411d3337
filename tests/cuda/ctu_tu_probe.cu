// ctu_tu_probe.cu -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
//
// Runs batches of transform-unit jobs through the CTU search driver's own job code (for_tu_tasks, tu_eval / tu_core,
// coeff_cost_serial of kvazaar_b200/csrc/ctu/*.h) and returns every output of every job, so that tests/test_ctu_tu_jobs.py
// can compare them unit by unit with the compiled reference.  One source, two builds:
//   * nvcc, sm_90a (make probe -> tests/cuda/libkvzctu_probe.so): one CTA of 128 threads per batch with the driver's
//     launch bounds and shared-memory state, so the jobs run on the CTA, warp and half-warp teams the driver deals them to;
//   * g++ -x c++ (tools/build_hostsim.sh -> tests/hostsim/libkvzctu_probe_host.so): the one-thread CTA of the host build.
// It lives outside kvazaar_b200/csrc so that the product library never contains it.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <vector>

#include "../../kvazaar_b200/csrc/ctu/ctu_frame.h"

using namespace kvzctu;

namespace {

constexpr int kMaxN = 1024;       // samples / levels per task slot (a 32x32 unit)
constexpr int kRefLen = 68;       // IntraRefs::top / left

// Per batch: int32 [4] = first task, number of tasks, leader_tid, unused.  Per task: int32 [8] = colour, log2 side, mode,
// scan, RDOQ's tr_depth, alternative (-1: tu_eval, 0: transform, 1: transform skip -- the split alternatives of a 4x4
// luma unit), unused x2.  Outputs per task: int32 [8] = has, ssd, tr_skip, team size, first thread of the team, unused x3.
struct ProbeArgs {
  const CtuTables *T;
  const CtuConfig *cfg;         // [batch]
  const int32_t *batch;         // [batch][4]
  const uint8_t *cabac;         // [batch][2][CTX_COUNT]: state->cabac (RDOQ's models), then the search models
  const void *refs;             // [batch][3 colours][top, left][kRefLen] unfiltered references, samples
  const int32_t *task;          // [task][8]
  const void *src;              // [task][kMaxN] source samples, row stride = the unit's side
  int fill;
  void *pred, *rec;             // [task][kMaxN] samples
  int16_t *q;                   // [task][kMaxN]
  int32_t *oi;                  // [task][8]
  uint64_t *cg_mask;            // [task]
  double *bits;                 // [task]
};

template <typename Pix> CTU_FN_NOINLINE void probe_batch(const ProbeArgs &a, int b, CtuST<Pix> *S)
{
  const int32_t *bt = a.batch + 4 * b;
  const int first = bt[0], ntasks = bt[1];
  const int32_t *task = a.task + 8 * first;
  const CtuConfig *cfg = a.cfg + b;
  // the whole shared state holds a known byte: a job that reads scratch it did not write sees it
  #pragma unroll 1
  for (int i = CTU_TID; i < (int)sizeof(CtuST<Pix>); i += CTU_NT) ((uint8_t *)S)[i] = (uint8_t)a.fill;
  CTU_SYNC();
  if (CTU_TID == 0) S->leader_tid = bt[2];
  sm_tables_load(&S->tb, a.T);
  #pragma unroll 1
  for (int i = CTU_TID; i < CTX_COUNT; i += CTU_NT) {
    S->cabac0.ctx[i] = a.cabac[(size_t)b * 2 * CTX_COUNT + i];
    S->sc.ctx[i] = a.cabac[(size_t)b * 2 * CTX_COUNT + CTX_COUNT + i];
  }
  if (CTU_TID == 0) S->sc.update = 0;
  // references of each colour the batch has (one unit size per colour, as in the driver's batches)
  int l2[3] = { 2, 2, 2 }, mask = 0;
  for (int t = 0; t < ntasks; ++t) { const int col = task[8 * t]; if (!((mask >> col) & 1)) { mask |= 1 << col; l2[col] = task[8 * t + 1]; } }
  const Pix *rin = (const Pix *)a.refs + (size_t)b * 3 * 2 * kRefLen;
  #pragma unroll 1
  for (int i = CTU_TID; i < 3 * kRefLen; i += CTU_NT) {
    const int col = i / kRefLen, e = i % kRefLen;
    if (!((mask >> col) & 1) || e > 2 * (1 << l2[col])) continue;
    S->refs[col].top[e] = rin[(col * 2 + 0) * kRefLen + e];
    S->refs[col].left[e] = rin[(col * 2 + 1) * kRefLen + e];
  }
  CTU_SYNC();
  refs_smooth_dc(l2, mask, (mask & 1) ? 2 * (1 << l2[0]) + 1 : 0, S->refs);
  const CtxT<Pix> c = { a.T, cfg, NULL, S };
  // the body of search_cu_intra's RDO batch (ctu_search.h), outputs kept per task
  for_tu_tasks(c, ntasks, [&](int t) { return tu_class(task[8 * t + 1], task[8 * t]); }, [&](const Team &tm, unsigned char *slot, int t) {
    const int32_t *d = task + 8 * t;
    const int col = d[0], log2n = d[1], n = 1 << log2n, alt = d[5];
    const size_t k = (size_t)(first + t);
    const TuS<Pix> tu = tu_at<Pix>(slot, n * n);
    TuJob<Pix> j = { &S->refs[col], (const Pix *)a.src + k * kMaxN, n, col, log2n, d[2], d[3], d[4] };
    int ts = 0;
    if (alt >= 0) tu_core(tm, &S->tb, &S->tb, cfg, S->cabac0.ctx, tu, j, alt == 1);
    else ts = tu_eval(tm, &S->tb, &S->tb, cfg, S->cabac0.ctx, &S->sc, tu, j);
    Pix *pred = (Pix *)a.pred + k * kMaxN, *rec = (Pix *)a.rec + k * kMaxN;
    int16_t *q = a.q + k * kMaxN;
    #pragma unroll 1
    for (int e = tm.tid; e < n * n; e += tm.nt) { pred[e] = tu.pred()[e]; rec[e] = tu.rec()[e]; q[e] = tu.q()[e]; }
    if (tm.tid == 0) {
      const TuFixed<Pix> *fx = tu.fx();
      const uint64_t m = (uint64_t)fx->cg_mask[0] | ((uint64_t)fx->cg_mask[1] << 32);
      int32_t *o = a.oi + 8 * k;
      o[0] = fx->has; o[1] = fx->ssd; o[2] = ts; o[3] = tm.nt; o[4] = CTU_TID - tm.tid;
      a.cg_mask[k] = m;
      a.bits[k] = fx->has ? coeff_cost_serial(&S->tb, &S->tb, cfg, &S->sc, tu.q(), log2n, col ? 2 : 0, d[3], 0, m) : 0.0;
    }
    tsync(tm);
  });
}

#if defined(__CUDACC__)
template <typename Pix> __global__ void __launch_bounds__(128, 3) probe_kernel(const __grid_constant__ ProbeArgs a)
{
  probe_batch<Pix>(a, blockIdx.x, reinterpret_cast<CtuST<Pix> *>(ctu_smem_raw));
}

#define PROBE_CHECK(expr) do { const cudaError_t e_ = (expr); if (e_ != cudaSuccess) { fprintf(stderr, "ctu_tu_probe: %s: %s\n", #expr, cudaGetErrorString(e_)); rc = -1; goto out; } } while (0)

template <typename Pix> int run(int nbatch, int ntask, ProbeArgs h)
{
  int rc = 0;
  const size_t pix = sizeof(Pix);
  std::vector<void *> bufs;
  bool ok = true;
  // device copies of the inputs; outputs are copied back below
  auto up = [&](const void *p, size_t bytes) -> void * {
    void *d = NULL;
    if (cudaMalloc(&d, bytes) != cudaSuccess) { ok = false; return NULL; }
    bufs.push_back(d);
    if (p && cudaMemcpy(d, p, bytes, cudaMemcpyHostToDevice) != cudaSuccess) ok = false;
    return d;
  };
  CtuTables tables;
  ctu_tables_init(&tables);
  ProbeArgs a = h;
  const size_t nt = (size_t)ntask;
  a.T = (const CtuTables *)up(&tables, sizeof(tables));
  a.cfg = (const CtuConfig *)up(h.cfg, nbatch * sizeof(CtuConfig));
  a.batch = (const int32_t *)up(h.batch, nbatch * 4 * sizeof(int32_t));
  a.cabac = (const uint8_t *)up(h.cabac, nbatch * 2 * CTX_COUNT);
  a.refs = up(h.refs, nbatch * 3 * 2 * kRefLen * pix);
  a.task = (const int32_t *)up(h.task, nt * 8 * sizeof(int32_t));
  a.src = up(h.src, nt * kMaxN * pix);
  a.pred = up(NULL, nt * kMaxN * pix);
  a.rec = up(NULL, nt * kMaxN * pix);
  a.q = (int16_t *)up(NULL, nt * kMaxN * 2);
  a.oi = (int32_t *)up(NULL, nt * 8 * sizeof(int32_t));
  a.cg_mask = (uint64_t *)up(NULL, nt * sizeof(uint64_t));
  a.bits = (double *)up(NULL, nt * sizeof(double));
  if (!ok) { fprintf(stderr, "ctu_tu_probe: device allocation or upload failed\n"); rc = -1; goto out; }
  PROBE_CHECK(cudaFuncSetAttribute(probe_kernel<Pix>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(CtuST<Pix>)));
  probe_kernel<Pix><<<nbatch, 128, sizeof(CtuST<Pix>)>>>(a);
  PROBE_CHECK(cudaGetLastError());
  PROBE_CHECK(cudaDeviceSynchronize());
  PROBE_CHECK(cudaMemcpy(h.pred, a.pred, nt * kMaxN * pix, cudaMemcpyDeviceToHost));
  PROBE_CHECK(cudaMemcpy(h.rec, a.rec, nt * kMaxN * pix, cudaMemcpyDeviceToHost));
  PROBE_CHECK(cudaMemcpy(h.q, a.q, nt * kMaxN * 2, cudaMemcpyDeviceToHost));
  PROBE_CHECK(cudaMemcpy(h.oi, a.oi, nt * 8 * sizeof(int32_t), cudaMemcpyDeviceToHost));
  PROBE_CHECK(cudaMemcpy(h.cg_mask, a.cg_mask, nt * sizeof(uint64_t), cudaMemcpyDeviceToHost));
  PROBE_CHECK(cudaMemcpy(h.bits, a.bits, nt * sizeof(double), cudaMemcpyDeviceToHost));
out:
  for (void *p : bufs) cudaFree(p);
  return rc;
}
#else
template <typename Pix> int run(int nbatch, int, ProbeArgs a)
{
  CtuTables *tables = new CtuTables;
  ctu_tables_init(tables);
  a.T = tables;
  CtuST<Pix> *S = (CtuST<Pix> *)malloc(sizeof(CtuST<Pix>));
  for (int b = 0; b < nbatch; ++b) probe_batch<Pix>(a, b, S);
  free(S);
  delete tables;
  return 0;
}
#endif

}  // namespace

extern "C" {

// Runs `nbatch` batches (one for_tu_tasks call each) of the `ntask` tasks; see ProbeArgs for the layouts.  Samples are
// uint8_t at bitdepth 8 and uint16_t at bitdepth 10.  Returns 0, or -1 on a bad argument or a CUDA error.
int kvz_ctu_probe_run(int bitdepth, int nbatch, const void *cfg, const int32_t *batch, const uint8_t *cabac, const void *refs, int ntask,
                      const int32_t *task, const void *src, int fill, void *pred, void *rec, int16_t *q, int32_t *oi, uint64_t *cg_mask, double *bits)
{
  if (nbatch <= 0 || ntask <= 0) return -1;
  for (int b = 0; b < nbatch; ++b) {
    const int32_t *bt = batch + 4 * b;
    if (bt[1] < 1 || bt[1] > 32 || bt[0] < 0 || bt[0] + bt[1] > ntask || (bt[2] & 31) || bt[2] < 0 || bt[2] > 96) return -1;
  }
  for (int t = 0; t < ntask; ++t) {
    const int32_t *d = task + 8 * t;
    if (d[0] < 0 || d[0] > 2 || d[1] < 2 || d[1] > (d[0] ? 4 : 5) || d[2] < 0 || d[2] > 34 || d[3] < 0 || d[3] > 2 || d[5] < -1 || d[5] > 1) return -1;
    if ((d[5] >= 0 && !(d[0] == 0 && d[1] == 2)) || (d[1] >= 4 && d[3] != 0)) return -1;   // 16x16 / 32x32: diagonal only
  }
  ProbeArgs a = { NULL, (const CtuConfig *)cfg, batch, cabac, refs, task, src, fill, pred, rec, q, oi, cg_mask, bits };
  if (bitdepth == 8) return run<uint8_t>(nbatch, ntask, a);
  if (bitdepth == 10) return run<uint16_t>(nbatch, ntask, a);
  return -1;
}

}  // extern "C"
