// me_search.cu -- integer motion estimation of a batch of PUs (SURVEY §8f rank 4): kvz_cuda_me_search_batch.
//
// One warp per PU.  The search is a chain of dependent decisions (every point's cost decides where the next one
// lies: search_inter.c:712-792), so the parallelism inside a PU is the SAD of one point -- its pixels spread over the
// 32 lanes, summed with shuffles -- and the parallelism of the launch is the PUs.  All decisions are warp-uniform
// (every lane holds the same best cost after the shuffle reduction), so there is no shared memory and no barrier.
// Bound: latency of ~20-40 dependent points per PU; the pixels of neighbouring points overlap and stay in L1/L2, the
// HBM traffic is one read of both pictures.
#include "common.cuh"
#include "me/me_search.h"
#include "me/me_cand.h"
#include "me/me_frac.h"
#include "me/me_merge.h"
#include "me/me_mc.h"

namespace {

constexpr int kWarpsPerCta = 4;

template <typename Pix, bool SATD_FINAL>
__global__ void __launch_bounds__(kWarpsPerCta * 32) me_search_kernel(kvz_cuda_me_params p, const Pix *__restrict__ cur, int cur_stride,
                                                                      const Pix *__restrict__ ref, int ref_stride,
                                                                      const kvz_cuda_me_pu *__restrict__ pus, int count,
                                                                      kvz_cuda_me_result *__restrict__ out)
{
  const int warp = threadIdx.x >> 5;
  const kvzme::Lanes ln = { (int)(threadIdx.x & 31), 32 };
  const kvzme::Planes<Pix> pl = { cur, ref, cur_stride, ref_stride };
  // whole warps leave together: the shuffles inside pu_sad always see 32 lanes
  for (int i = blockIdx.x * kWarpsPerCta + warp; i < count; i += gridDim.x * kWarpsPerCta) {
    const kvz_cuda_me_pu pu = pus[i];
    if (SATD_FINAL) kvzme::search_pu_satd_final<Pix>(ln, p, pu, pl, &out[i]);      // cfg.fme_level == 0
    else kvzme::search_pu<Pix>(ln, p, pu, pl, &out[i]);
  }
}

// fractional search: one warp per PU, every lane interpolates and transforms the sub-blocks of its share in registers
template <typename Pix>
__global__ void __launch_bounds__(kWarpsPerCta * 32) me_frac_kernel(kvz_cuda_me_params p, int levels, const Pix *__restrict__ cur, int cur_stride,
                                                                    const Pix *__restrict__ ref, int ref_stride,
                                                                    const kvz_cuda_me_pu *__restrict__ pus, int count,
                                                                    kvz_cuda_me_result *__restrict__ out)
{
  const int warp = threadIdx.x >> 5;
  const kvzme::Lanes ln = { (int)(threadIdx.x & 31), 32 };
  const kvzme::Planes<Pix> pl = { cur, ref, cur_stride, ref_stride };
  for (int i = blockIdx.x * kWarpsPerCta + warp; i < count; i += gridDim.x * kWarpsPerCta) {
    const kvz_cuda_me_pu pu = pus[i];
    kvzme::frac_search_pu<Pix>(ln, p, pu, pl, levels, &out[i]);
  }
}

// merge analysis: one warp per PU, per accepted candidate one in-register prediction (one or two lists) + Hadamard cost
template <typename Pix>
__global__ void __launch_bounds__(kWarpsPerCta * 32) me_merge_kernel(kvz_cuda_me_params p, kvz_cuda_me_refs rf, const Pix *__restrict__ cur, int cur_stride,
                                                                     const kvz_cuda_me_pu *__restrict__ pus, int count,
                                                                     kvz_cuda_me_merge_cost *__restrict__ out)
{
  const int warp = threadIdx.x >> 5;
  const kvzme::Lanes ln = { (int)(threadIdx.x & 31), 32 };
  const kvzme::Planes<Pix> pl = { cur, nullptr, cur_stride, 0 };
  kvzme::RefSet<Pix> rs;
  for (int i = 0; i < 16; ++i) { rs.plane[i] = (const Pix *)rf.plane[i]; rs.stride[i] = rf.stride[i]; }
  for (int i = blockIdx.x * kWarpsPerCta + warp; i < count; i += gridDim.x * kWarpsPerCta) {
    const kvz_cuda_me_pu pu = pus[i];
    kvzme::merge_cost_pu<Pix>(ln, p, rf, rs, pu, pl, &out[i]);
  }
}

// bi-prediction from two uni-predictions: one warp per PU
template <typename Pix>
__global__ void __launch_bounds__(kWarpsPerCta * 32) me_bipred_kernel(kvz_cuda_me_params p, kvz_cuda_me_refs rf, const Pix *__restrict__ cur, int cur_stride,
                                                                      const kvz_cuda_me_bipred_pu *__restrict__ pus, int count,
                                                                      kvz_cuda_me_bipred_result *__restrict__ out)
{
  const int warp = threadIdx.x >> 5;
  const kvzme::Lanes ln = { (int)(threadIdx.x & 31), 32 };
  const kvzme::Planes<Pix> pl = { cur, nullptr, cur_stride, 0 };
  kvzme::RefSet<Pix> rs;
  for (int i = 0; i < 16; ++i) { rs.plane[i] = (const Pix *)rf.plane[i]; rs.stride[i] = rf.stride[i]; }
  for (int i = blockIdx.x * kWarpsPerCta + warp; i < count; i += gridDim.x * kWarpsPerCta) {
    const kvz_cuda_me_bipred_pu bp = pus[i];
    kvzme::bipred_pu<Pix>(ln, p, rf, rs, bp, pl, &out[i]);
  }
}

// motion compensation: one warp per PU, every lane writes the blocks of its share
template <typename Pix>
__global__ void __launch_bounds__(kWarpsPerCta * 32) me_predict_kernel(kvz_cuda_me_params p, kvz_cuda_me_mc_refs rf, const kvz_cuda_me_mc_pu *__restrict__ pus, int count,
                                                                       Pix *__restrict__ out_y, Pix *__restrict__ out_u, Pix *__restrict__ out_v)
{
  const int warp = threadIdx.x >> 5;
  const kvzme::Lanes ln = { (int)(threadIdx.x & 31), 32 };
  kvzme::McRefs<Pix> rs;
  for (int i = 0; i < 16; ++i) { rs.y[i] = (const Pix *)rf.y[i]; rs.u[i] = (const Pix *)rf.u[i]; rs.v[i] = (const Pix *)rf.v[i]; }
  for (int i = blockIdx.x * kWarpsPerCta + warp; i < count; i += gridDim.x * kWarpsPerCta) {
    const kvz_cuda_me_mc_pu pu = pus[i];
    kvzme::predict_pu<Pix>(ln, p, rf, rs, pu, out_y, out_u, out_v);
  }
}

// AMVP / merge candidates: one thread per PU, integer logic over the CU records (12-byte records, read through L1/L2)
__global__ void __launch_bounds__(128) me_cand_kernel(kvz_cuda_me_frame f, const kvz_cuda_me_cu *__restrict__ cus, int cu_stride,
                                                      const kvz_cuda_me_cu *__restrict__ col_cus, int col_stride,
                                                      const kvz_cuda_me_cand_pu *__restrict__ pus, int count, kvz_cuda_me_cand_out *__restrict__ out)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  const kvzme::CuImage cur = { cus, cu_stride }, col = { col_cus, col_stride };
  const kvz_cuda_me_cand_pu pu = pus[i];
  kvzme::candidates_of_pu(f, cur, col, pu, &out[i]);
}

int check_args(const kvz_cuda_me_params *p, const void *cur, int cur_stride, const void *ref, int ref_stride, const void *pus, int count,
               const void *out)
{
  KVZC_ARG(p && cur && ref && count >= 0 && (count == 0 || (pus && out)));
  KVZC_ARG(kvzme::params_supported(*p) == 0);
  KVZC_ARG(cur_stride >= p->width && ref_stride >= p->width);
  return 0;
}

}  // namespace

extern "C" int kvz_cuda_me_params_supported(const kvz_cuda_me_params *p) { return p ? kvzme::params_supported(*p) : -1; }

extern "C" int kvz_cuda_me_search_batch(const kvz_cuda_me_params *p, const void *cur_dev, int cur_stride, const void *ref_dev, int ref_stride,
                                        const kvz_cuda_me_pu *pus_dev, int count, kvz_cuda_me_result *out_dev, void *stream)
{
  KVZC_REQUIRE_DEVICE();
  if (int e = check_args(p, cur_dev, cur_stride, ref_dev, ref_stride, pus_dev, count, out_dev)) return e;
  if (count == 0) return 0;
  const int ctas = (count + kWarpsPerCta - 1) / kWarpsPerCta;
  const int cap = kvzc::g_sm_count > 0 ? kvzc::g_sm_count * 16 : 132 * 16;     // 16 CTAs of 4 warps per SM; more PUs loop
  const int grid = ctas < cap ? ctas : cap;
  const cudaStream_t st = kvzc::as_stream(stream);
  const dim3 block(kWarpsPerCta * 32);
  const uint8_t *c8 = (const uint8_t *)cur_dev, *r8 = (const uint8_t *)ref_dev;
  const uint16_t *c16 = (const uint16_t *)cur_dev, *r16 = (const uint16_t *)ref_dev;
  if (p->bitdepth == 8 && !p->satd_final) me_search_kernel<uint8_t, false><<<grid, block, 0, st>>>(*p, c8, cur_stride, r8, ref_stride, pus_dev, count, out_dev);
  else if (p->bitdepth == 8) me_search_kernel<uint8_t, true><<<grid, block, 0, st>>>(*p, c8, cur_stride, r8, ref_stride, pus_dev, count, out_dev);
  else if (!p->satd_final) me_search_kernel<uint16_t, false><<<grid, block, 0, st>>>(*p, c16, cur_stride, r16, ref_stride, pus_dev, count, out_dev);
  else me_search_kernel<uint16_t, true><<<grid, block, 0, st>>>(*p, c16, cur_stride, r16, ref_stride, pus_dev, count, out_dev);
  KVZC_LAUNCHED();
  return 0;
}

// host buffers, synchronous: the binding a host that keeps its pictures in host memory would call
extern "C" int kvz_cuda_call_me_search(const kvz_cuda_me_params *p, const void *cur, int cur_stride, const void *ref, int ref_stride,
                                       const kvz_cuda_me_pu *pus, int count, kvz_cuda_me_result *out)
{
  KVZC_REQUIRE_DEVICE();
  if (int e = check_args(p, cur, cur_stride, ref, ref_stride, pus, count, out)) return e;
  if (count == 0) return 0;
  const size_t px = p->bitdepth == 8 ? 1 : 2;
  const size_t cur_bytes = (size_t)cur_stride * p->height * px, ref_bytes = (size_t)ref_stride * p->height * px;
  const size_t pu_bytes = (size_t)count * sizeof(kvz_cuda_me_pu), out_bytes = (size_t)count * sizeof(kvz_cuda_me_result);
  uint8_t *d = nullptr;
  const size_t o_ref = (cur_bytes + 255) & ~(size_t)255, o_pu = (o_ref + ref_bytes + 255) & ~(size_t)255, o_out = (o_pu + pu_bytes + 255) & ~(size_t)255;
  KVZC_CHECK(cudaMalloc(&d, o_out + out_bytes));
  cudaStream_t st = nullptr;
  int rc = 0;
  cudaError_t e = cudaMemcpyAsync(d, cur, cur_bytes, cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess) e = cudaMemcpyAsync(d + o_ref, ref, ref_bytes, cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess) e = cudaMemcpyAsync(d + o_pu, pus, pu_bytes, cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess)
    rc = kvz_cuda_me_search_batch(p, d, cur_stride, d + o_ref, ref_stride, (const kvz_cuda_me_pu *)(d + o_pu), count, (kvz_cuda_me_result *)(d + o_out), st);
  if (e == cudaSuccess && rc == 0) e = cudaMemcpyAsync(out, d + o_out, out_bytes, cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess && rc == 0) e = cudaStreamSynchronize(st);
  cudaFree(d);
  if (e != cudaSuccess) { kvzc::set_error("kvz_cuda_call_me_search: %s", cudaGetErrorString(e)); return KVZ_CUDA_E_RUNTIME; }
  return rc;
}

extern "C" int kvz_cuda_me_candidates_batch(const kvz_cuda_me_frame *f, const kvz_cuda_me_cu *cus_dev, int cu_stride, const kvz_cuda_me_cu *col_cus_dev,
                                            int col_stride, const kvz_cuda_me_cand_pu *pus_dev, int count, kvz_cuda_me_cand_out *out_dev, void *stream)
{
  KVZC_REQUIRE_DEVICE();
  KVZC_ARG(f && cus_dev && col_cus_dev && count >= 0 && (count == 0 || (pus_dev && out_dev)));
  KVZC_ARG(kvzme::frame_supported(*f) == 0);
  KVZC_ARG(cu_stride >= (f->width + 3) / 4 && col_stride >= (f->width + 3) / 4);
  if (count == 0) return 0;
  me_cand_kernel<<<(count + 127) / 128, 128, 0, kvzc::as_stream(stream)>>>(*f, cus_dev, cu_stride, col_cus_dev, col_stride, pus_dev, count, out_dev);
  KVZC_LAUNCHED();
  return 0;
}

extern "C" int kvz_cuda_call_me_candidates(const kvz_cuda_me_frame *f, const kvz_cuda_me_cu *cus, int cu_stride, const kvz_cuda_me_cu *col_cus,
                                           int col_stride, int cu_rows, const kvz_cuda_me_cand_pu *pus, int count, kvz_cuda_me_cand_out *out)
{
  KVZC_REQUIRE_DEVICE();
  KVZC_ARG(f && cus && col_cus && cu_rows > 0 && count >= 0 && (count == 0 || (pus && out)));
  if (count == 0) return 0;
  const size_t cu_bytes = (size_t)cu_stride * cu_rows * sizeof(kvz_cuda_me_cu), col_bytes = (size_t)col_stride * cu_rows * sizeof(kvz_cuda_me_cu);
  const size_t pu_bytes = (size_t)count * sizeof(kvz_cuda_me_cand_pu), out_bytes = (size_t)count * sizeof(kvz_cuda_me_cand_out);
  const size_t o_col = (cu_bytes + 255) & ~(size_t)255, o_pu = (o_col + col_bytes + 255) & ~(size_t)255, o_out = (o_pu + pu_bytes + 255) & ~(size_t)255;
  uint8_t *d = nullptr;
  KVZC_CHECK(cudaMalloc(&d, o_out + out_bytes));
  cudaStream_t st = nullptr;
  int rc = 0;
  cudaError_t e = cudaMemcpyAsync(d, cus, cu_bytes, cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess) e = cudaMemcpyAsync(d + o_col, col_cus, col_bytes, cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess) e = cudaMemcpyAsync(d + o_pu, pus, pu_bytes, cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess)
    rc = kvz_cuda_me_candidates_batch(f, (const kvz_cuda_me_cu *)d, cu_stride, (const kvz_cuda_me_cu *)(d + o_col), col_stride,
                                      (const kvz_cuda_me_cand_pu *)(d + o_pu), count, (kvz_cuda_me_cand_out *)(d + o_out), st);
  if (e == cudaSuccess && rc == 0) e = cudaMemcpyAsync(out, d + o_out, out_bytes, cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess && rc == 0) e = cudaStreamSynchronize(st);
  cudaFree(d);
  if (e != cudaSuccess) { kvzc::set_error("kvz_cuda_call_me_candidates: %s", cudaGetErrorString(e)); return KVZ_CUDA_E_RUNTIME; }
  return rc;
}

extern "C" int kvz_cuda_me_frac_search_batch(const kvz_cuda_me_params *p, int fme_level, const void *cur_dev, int cur_stride, const void *ref_dev,
                                             int ref_stride, const kvz_cuda_me_pu *pus_dev, int count, kvz_cuda_me_result *out_dev, void *stream)
{
  KVZC_REQUIRE_DEVICE();
  if (int e = check_args(p, cur_dev, cur_stride, ref_dev, ref_stride, pus_dev, count, out_dev)) return e;
  KVZC_ARG(fme_level >= 1 && fme_level <= 4);
  if (count == 0) return 0;
  const int ctas = (count + kWarpsPerCta - 1) / kWarpsPerCta;
  const int cap = kvzc::g_sm_count > 0 ? kvzc::g_sm_count * 16 : 132 * 16;
  const int grid = ctas < cap ? ctas : cap;
  if (p->bitdepth == 8)
    me_frac_kernel<uint8_t><<<grid, kWarpsPerCta * 32, 0, kvzc::as_stream(stream)>>>(*p, fme_level, (const uint8_t *)cur_dev, cur_stride,
                                                                                  (const uint8_t *)ref_dev, ref_stride, pus_dev, count, out_dev);
  else
    me_frac_kernel<uint16_t><<<grid, kWarpsPerCta * 32, 0, kvzc::as_stream(stream)>>>(*p, fme_level, (const uint16_t *)cur_dev, cur_stride,
                                                                                   (const uint16_t *)ref_dev, ref_stride, pus_dev, count, out_dev);
  KVZC_LAUNCHED();
  return 0;
}

extern "C" int kvz_cuda_call_me_frac_search(const kvz_cuda_me_params *p, int fme_level, const void *cur, int cur_stride, const void *ref,
                                            int ref_stride, const kvz_cuda_me_pu *pus, int count, kvz_cuda_me_result *out)
{
  KVZC_REQUIRE_DEVICE();
  if (int e = check_args(p, cur, cur_stride, ref, ref_stride, pus, count, out)) return e;
  if (count == 0) return 0;
  const size_t px = p->bitdepth == 8 ? 1 : 2;
  const size_t cur_bytes = (size_t)cur_stride * p->height * px, ref_bytes = (size_t)ref_stride * p->height * px;
  const size_t pu_bytes = (size_t)count * sizeof(kvz_cuda_me_pu), out_bytes = (size_t)count * sizeof(kvz_cuda_me_result);
  uint8_t *d = nullptr;
  const size_t o_ref = (cur_bytes + 255) & ~(size_t)255, o_pu = (o_ref + ref_bytes + 255) & ~(size_t)255, o_out = (o_pu + pu_bytes + 255) & ~(size_t)255;
  KVZC_CHECK(cudaMalloc(&d, o_out + out_bytes));
  cudaStream_t st = nullptr;
  int rc = 0;
  cudaError_t e = cudaMemcpyAsync(d, cur, cur_bytes, cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess) e = cudaMemcpyAsync(d + o_ref, ref, ref_bytes, cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess) e = cudaMemcpyAsync(d + o_pu, pus, pu_bytes, cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess)
    rc = kvz_cuda_me_frac_search_batch(p, fme_level, d, cur_stride, d + o_ref, ref_stride, (const kvz_cuda_me_pu *)(d + o_pu), count,
                                       (kvz_cuda_me_result *)(d + o_out), st);
  if (e == cudaSuccess && rc == 0) e = cudaMemcpyAsync(out, d + o_out, out_bytes, cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess && rc == 0) e = cudaStreamSynchronize(st);
  cudaFree(d);
  if (e != cudaSuccess) { kvzc::set_error("kvz_cuda_call_me_frac_search: %s", cudaGetErrorString(e)); return KVZ_CUDA_E_RUNTIME; }
  return rc;
}

extern "C" int kvz_cuda_me_merge_cost_batch(const kvz_cuda_me_params *p, const kvz_cuda_me_refs *refs, const void *cur_dev, int cur_stride,
                                            const kvz_cuda_me_pu *pus_dev, int count, kvz_cuda_me_merge_cost *out_dev, void *stream)
{
  KVZC_REQUIRE_DEVICE();
  KVZC_ARG(p && refs && cur_dev && count >= 0 && (count == 0 || (pus_dev && out_dev)));
  KVZC_ARG(kvzme::params_supported(*p) == 0 && cur_stride >= p->width);
  for (int l = 0; l < 2; ++l)
    for (int i = 0; i < 16; ++i) KVZC_ARG(refs->ref_LX[l][i] < 16);
  if (count == 0) return 0;
  const int ctas = (count + kWarpsPerCta - 1) / kWarpsPerCta;
  const int cap = kvzc::g_sm_count > 0 ? kvzc::g_sm_count * 16 : 132 * 16;
  const int grid = ctas < cap ? ctas : cap;
  if (p->bitdepth == 8)
    me_merge_kernel<uint8_t><<<grid, kWarpsPerCta * 32, 0, kvzc::as_stream(stream)>>>(*p, *refs, (const uint8_t *)cur_dev, cur_stride, pus_dev, count, out_dev);
  else
    me_merge_kernel<uint16_t><<<grid, kWarpsPerCta * 32, 0, kvzc::as_stream(stream)>>>(*p, *refs, (const uint16_t *)cur_dev, cur_stride, pus_dev, count, out_dev);
  KVZC_LAUNCHED();
  return 0;
}

extern "C" int kvz_cuda_me_bipred_batch(const kvz_cuda_me_params *p, const kvz_cuda_me_refs *refs, const void *cur_dev, int cur_stride,
                                        const kvz_cuda_me_bipred_pu *pus_dev, int count, kvz_cuda_me_bipred_result *out_dev, void *stream)
{
  KVZC_REQUIRE_DEVICE();
  KVZC_ARG(p && refs && cur_dev && count >= 0 && (count == 0 || (pus_dev && out_dev)));
  KVZC_ARG(kvzme::params_supported(*p) == 0 && cur_stride >= p->width);
  for (int l = 0; l < 2; ++l)
    for (int i = 0; i < 16; ++i) KVZC_ARG(refs->ref_LX[l][i] < 16);
  if (count == 0) return 0;
  const int ctas = (count + kWarpsPerCta - 1) / kWarpsPerCta;
  const int cap = kvzc::g_sm_count > 0 ? kvzc::g_sm_count * 16 : 132 * 16;
  const int grid = ctas < cap ? ctas : cap;
  if (p->bitdepth == 8)
    me_bipred_kernel<uint8_t><<<grid, kWarpsPerCta * 32, 0, kvzc::as_stream(stream)>>>(*p, *refs, (const uint8_t *)cur_dev, cur_stride, pus_dev, count, out_dev);
  else
    me_bipred_kernel<uint16_t><<<grid, kWarpsPerCta * 32, 0, kvzc::as_stream(stream)>>>(*p, *refs, (const uint16_t *)cur_dev, cur_stride, pus_dev, count, out_dev);
  KVZC_LAUNCHED();
  return 0;
}

extern "C" int kvz_cuda_me_predict_batch(const kvz_cuda_me_params *p, const kvz_cuda_me_mc_refs *refs, const kvz_cuda_me_mc_pu *pus_dev, int count,
                                         void *pred_y_dev, void *pred_u_dev, void *pred_v_dev, void *stream)
{
  KVZC_REQUIRE_DEVICE();
  KVZC_ARG(p && refs && count >= 0 && (count == 0 || (pus_dev && pred_y_dev && pred_u_dev && pred_v_dev)));
  KVZC_ARG(kvzme::params_supported(*p) == 0 && (p->width & 1) == 0 && (p->height & 1) == 0);
  for (int l = 0; l < 2; ++l)
    for (int i = 0; i < 16; ++i) KVZC_ARG(refs->ref_LX[l][i] < 16);
  for (int i = 0; i < 16; ++i) KVZC_ARG((refs->y[i] == nullptr) == (refs->u[i] == nullptr) && (refs->y[i] == nullptr) == (refs->v[i] == nullptr));
  if (count == 0) return 0;
  const int ctas = (count + kWarpsPerCta - 1) / kWarpsPerCta;
  const int cap = kvzc::g_sm_count > 0 ? kvzc::g_sm_count * 16 : 132 * 16;
  const int grid = ctas < cap ? ctas : cap;
  if (p->bitdepth == 8)
    me_predict_kernel<uint8_t><<<grid, kWarpsPerCta * 32, 0, kvzc::as_stream(stream)>>>(*p, *refs, pus_dev, count, (uint8_t *)pred_y_dev, (uint8_t *)pred_u_dev, (uint8_t *)pred_v_dev);
  else
    me_predict_kernel<uint16_t><<<grid, kWarpsPerCta * 32, 0, kvzc::as_stream(stream)>>>(*p, *refs, pus_dev, count, (uint16_t *)pred_y_dev, (uint16_t *)pred_u_dev, (uint16_t *)pred_v_dev);
  KVZC_LAUNCHED();
  return 0;
}
