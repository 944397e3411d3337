// intra.cu -- intra group: batched prediction, reference building and the entry point of the fused frame-level rough
// search (rough_search.cu).
#include "common.cuh"
#include "intra.cuh"

namespace kvzc {

// ---------------------------------------------------------------------------------------------
// Batched prediction: CTA of 256 threads handles G = max(1, 256 / w^2) blocks, thread per pixel.
// ---------------------------------------------------------------------------------------------
template <class T>
__global__ void __launch_bounds__(256) intra_predict_kernel(int level, int log2w, int color, int filter_boundary,
                                                            const T *__restrict__ ref_top, const T *__restrict__ ref_left,
                                                            const int8_t *__restrict__ modes, int count,
                                                            T *__restrict__ dst, int g_per_cta)
{
  __shared__ T s_ref[16][4][65];      // [block in CTA][top,left,ftop,fleft][entry]
  __shared__ int s_dc[16];
  const int w = 1 << log2w, n = 2 * w + 1, ww = w * w;
  const int first = blockIdx.x * g_per_cta;
  const int g = min(g_per_cta, count - first);
  for (int e = threadIdx.x; e < g * 2 * n; e += blockDim.x) {
    const int b = e / (2 * n), r = e - b * 2 * n, which = r / n, i = r - which * n;
    s_ref[b][which][i] = (which ? ref_left : ref_top)[(size_t)(first + b) * n + i];
  }
  __syncthreads();
  for (int e = threadIdx.x; e < g * 2 * n; e += blockDim.x) {
    const int b = e / (2 * n), r = e - b * 2 * n, which = r / n, i = r - which * n;
    s_ref[b][2 + which][i] = (T)filter_ref_entry(s_ref[b][0], s_ref[b][1], which == 0, i, n);
  }
  if (threadIdx.x < g) s_dc[threadIdx.x] = dc_value(log2w, s_ref[threadIdx.x][0], s_ref[threadIdx.x][1]);
  __syncthreads();
  for (int e = threadIdx.x; e < g * ww; e += blockDim.x) {
    const int b = e / ww, r = e - b * ww, y = r >> log2w, x = r & (w - 1);
    const int mode = modes[first + b];
    const T *top = s_ref[b][0], *left = s_ref[b][1];
    int v;
    if (level == 0) {
      if (mode == 0) v = planar_px(log2w, top, left, x, y);
      else if (mode == 1) v = filtered_dc_px(top, left, s_dc[b], x, y);
      else v = angular_px(mode, top, left, x, y);
    } else {
      v = intra_predict_px(log2w, mode, color, filter_boundary != 0, top, left, s_ref[b][2], s_ref[b][3], s_dc[b], x, y);
    }
    dst[(size_t)(first + b) * ww + r] = (T)v;
  }
}

// kvz_intra_build_reference over a frame plane: one warp per block
template <class T>
__global__ void __launch_bounds__(128) build_reference_kernel(int log2w, int color, const T *__restrict__ rec, int stride,
                                                              int pic_w, int pic_h, const int32_t *__restrict__ xy,
                                                              int count, T *__restrict__ out_top, T *__restrict__ out_left)
{
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= count) return;
  const int n = 2 * (1 << log2w) + 1;
  const BuildRefCtx c = build_ref_ctx(log2w, color, xy[2 * warp], xy[2 * warp + 1], pic_w, pic_h);
  for (int i = lane; i < n; i += 32) {
    out_top[(size_t)warp * n + i] = (T)build_ref_entry(c, rec, stride, true, i);
    out_left[(size_t)warp * n + i] = (T)build_ref_entry(c, rec, stride, false, i);
  }
}

}  // namespace kvzc

using namespace kvzc;

namespace kvzc {
int rough_search_u8(int log2w, const uint8_t *src, const uint8_t *rec, int stride, int pic_w, int pic_h, uint32_t *costs,
                    int8_t *best_mode, uint32_t *best_cost, cudaStream_t st);
int rough_search_u16(int log2w, const uint16_t *src, const uint16_t *rec, int stride, int pic_w, int pic_h, uint32_t *costs,
                     int8_t *best_mode, uint32_t *best_cost, cudaStream_t st);
}

extern "C" {

int kvz_cuda_intra_predict_batch(int level, int log2_width, int color, int filter_boundary, int bitdepth,
                                 const void *ref_top, const void *ref_left, const int8_t *modes, int count, void *dst,
                                 void *stream)
{
  KVZC_REQUIRE_DEVICE();
  KVZC_ARG(ref_top && ref_left && modes && dst && log2_width >= 2 && log2_width <= 5 && (level == 0 || level == 1));
  if (count == 0) return 0;
  const int ww = 1 << (2 * log2_width);
  const int g = ww >= 256 ? 1 : 256 / ww;
  const int grid = (count + g - 1) / g;
  if (bitdepth == 8)
    intra_predict_kernel<uint8_t><<<grid, 256, 0, as_stream(stream)>>>(level, log2_width, color, filter_boundary, (const uint8_t *)ref_top, (const uint8_t *)ref_left, modes, count, (uint8_t *)dst, g);
  else
    intra_predict_kernel<uint16_t><<<grid, 256, 0, as_stream(stream)>>>(level, log2_width, color, filter_boundary, (const uint16_t *)ref_top, (const uint16_t *)ref_left, modes, count, (uint16_t *)dst, g);
  KVZC_LAUNCHED();
  return 0;
}

int kvz_cuda_intra_build_reference_batch(int log2_width, int color, int bitdepth, const void *rec_plane, int stride,
                                         int pic_w, int pic_h, const int32_t *luma_xy, int count, void *out_top,
                                         void *out_left, void *stream)
{
  KVZC_REQUIRE_DEVICE();
  KVZC_ARG(rec_plane && luma_xy && out_top && out_left && log2_width >= 2 && log2_width <= 5 && color >= 0 && color <= 2);
  if (count == 0) return 0;
  const int grid = (count * 32 + 127) / 128;
  if (bitdepth == 8)
    build_reference_kernel<uint8_t><<<grid, 128, 0, as_stream(stream)>>>(log2_width, color, (const uint8_t *)rec_plane, stride, pic_w, pic_h, luma_xy, count, (uint8_t *)out_top, (uint8_t *)out_left);
  else
    build_reference_kernel<uint16_t><<<grid, 128, 0, as_stream(stream)>>>(log2_width, color, (const uint16_t *)rec_plane, stride, pic_w, pic_h, luma_xy, count, (uint16_t *)out_top, (uint16_t *)out_left);
  KVZC_LAUNCHED();
  return 0;
}

int kvz_cuda_intra_rough_search_frame(int log2_width, int bitdepth, const void *src_plane, const void *rec_plane,
                                      int stride, int pic_w, int pic_h, uint32_t *costs, void *stream)
{
  KVZC_REQUIRE_DEVICE();
  KVZC_ARG(src_plane && rec_plane && costs && log2_width >= 2 && log2_width <= 5 && pic_w % 8 == 0 && pic_h % 8 == 0);
  if (bitdepth == 8)
    return rough_search_u8(log2_width, (const uint8_t *)src_plane, (const uint8_t *)rec_plane, stride, pic_w, pic_h, costs, nullptr, nullptr, as_stream(stream));
  return rough_search_u16(log2_width, (const uint16_t *)src_plane, (const uint16_t *)rec_plane, stride, pic_w, pic_h, costs, nullptr, nullptr, as_stream(stream));
}

}  // extern "C"
