// ipol.cu -- ipol group: fractional sample interpolation (8-tap luma / 4-tap chroma), the four
// fractional-motion-estimation filter stages and border extension.
// Reference: src/strategies/generic/ipol-generic.c; FIR taps src/filter.c:66-84.
#include "common.cuh"

namespace kvzc {

static __constant__ int8_t c_luma_fir[4][8] = {
  { 0, 0, 0, 64, 0, 0, 0, 0 }, { -1, 4, -10, 58, 17, -5, 1, 0 }, { -1, 4, -11, 40, 40, -11, 4, -1 }, { 0, 1, -5, 17, 58, -10, 4, -1 } };
static __constant__ int8_t c_chroma_fir[8][4] = {
  { 0, 64, 0, 0 }, { -2, 58, 10, -2 }, { -4, 54, 16, -2 }, { -6, 46, 28, -4 },
  { -4, 36, 36, -4 }, { -4, 28, 46, -6 }, { -2, 16, 54, -4 }, { -2, 10, 58, -2 } };

template <class T> __device__ __forceinline__ int clip_pix(int v) { return clip3(0, (1 << PixTraits<T>::bd) - 1, v); }

// sample_quarterpel_luma(_hi) / sample_octpel_chroma(_hi) (ref: ipol-generic.c:134-211, 681-758): one CTA per block.
// Horizontal pass into shared int16 rows, then vertical pass; intermediate truncation to int16 as in the reference.
template <class T>
__global__ void __launch_bounds__(256) sample_kernel(int kind, const T *__restrict__ src_plane, int src_stride,
                                                     void *__restrict__ dst_base, int dst_stride,
                                                     const kvz_cuda_ipol *__restrict__ descs)
{
  constexpr int BITS = PixTraits<T>::bd;
  __shared__ int16_t s_h[(64 + 7) * 64];
  const kvz_cuda_ipol d = descs[blockIdx.x];
  const bool chroma = kind >= KVZ_CUDA_IPOL_CHROMA, hi = kind & 1;
  const int taps = chroma ? 4 : 8, off = taps / 2 - 1;
  const int8_t *hf = chroma ? c_chroma_fir[d.mvx & 7] : c_luma_fir[d.mvx & 3];
  const int8_t *vf = chroma ? c_chroma_fir[d.mvy & 7] : c_luma_fir[d.mvy & 3];
  const T *src = src_plane + d.off_src;
  const int w = d.w, h = d.h;
  const int shift1 = BITS - 8, shift2 = 6, wp_shift = 14 - BITS, wp_off = 1 << (wp_shift - 1);
  for (int i = threadIdx.x; i < (h + taps - 1) * w; i += blockDim.x) {
    const int y = i / w, x = i - y * w;
    const T *p = src + (long)(y - off) * src_stride + (x - off);
    int t = 0;
    for (int k = 0; k < taps; ++k) t += hf[k] * (int)p[k];
    s_h[y * 64 + x] = (int16_t)(t >> shift1);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < h * w; i += blockDim.x) {
    const int y = i / w, x = i - y * w;
    int t = 0;
    for (int k = 0; k < taps; ++k) t += vf[k] * (int)s_h[(y + k) * 64 + x];
    t >>= shift2;
    if (hi) ((int16_t *)dst_base)[d.off_dst + (long)y * dst_stride + x] = (int16_t)t;
    else ((T *)dst_base)[d.off_dst + (long)y * dst_stride + x] = (T)clip_pix<T>((t + wp_off) >> wp_shift);
  }
}

// ---- FME filter stages (ref: ipol-generic.c:213-679) -------------------------------------------------------
// Shared state between the stages (all per block, in global memory because it is part of the interface):
//   im[k][y*64 + x]: horizontal 8-tap of phase k (im0: 0, im1: 2/4, im3: left qpel, im4: right qpel) of source row
//                    y - 3, window starting at column x - 2;  col[k][y]: same filter for the window at column -3.
// Every output is  clip(((int16)(vertical_tap_sum >> 6) + 32) >> 6)  for 8-bit.
template <class T> __device__ __forceinline__ int fme_round(int16_t s)
{
  constexpr int BITS = PixTraits<T>::bd;
  const int wp_shift = 14 - BITS, wp_off = 1 << (wp_shift - 1);
  return clip_pix<T>(((int)s + wp_off) >> wp_shift);
}
template <class T> __device__ __forceinline__ int fir8_px(const int8_t *f, const T *p, long st)
{ int t = 0;
#pragma unroll
  for (int k = 0; k < 8; ++k) t += f[k] * (int)p[k * st]; return t; }
__device__ __forceinline__ int fir8_im(const int8_t *f, const int16_t *p, int st)
{ int t = 0;
#pragma unroll
  for (int k = 0; k < 8; ++k) t += f[k] * (int)p[k * st]; return t; }

template <class T>
__device__ void fme_hor(const T *src, int ss, int w, int rows, int first_y, const int8_t *f, int16_t *im_k, int16_t *col_k)
{
  constexpr int shift1 = PixTraits<T>::bd - 8;
  for (int i = threadIdx.x; i < (rows - first_y) * (w + 1); i += blockDim.x) {
    const int y = first_y + i / (w + 1), x = i % (w + 1) - 1;       // x = -1 is the "first column" array
    const int v = fir8_px<T>(f, src + (long)(y - 3) * ss + (x < 0 ? -3 : x - 2), 1) >> shift1;
    if (x < 0) col_k[y] = (int16_t)v; else im_k[y * 64 + x] = (int16_t)v;
  }
}
template <class T>
__device__ void fme_ver_plane(T *out, int w, int h, const int8_t *vf, const int16_t *im_k, const int16_t *col_k,
                              int use_col, int yoff)
{
  for (int i = threadIdx.x; i < w * h; i += blockDim.x) {
    const int y = i / w, x = i - y * w;
    int16_t s;
    if (use_col && x == 0) s = (int16_t)(fir8_im(vf, col_k + y + yoff, 1) >> 6);
    else s = (int16_t)(fir8_im(vf, im_k + (y + yoff) * 64 + x - use_col, 64) >> 6);
    out[y * 64 + x] = (T)fme_round<T>(s);
  }
}

template <class T>
__global__ void __launch_bounds__(256) fme_kernel(int stage, const T *__restrict__ src_plane, int ss,
                                                  const int32_t *__restrict__ src_off, int w, int h,
                                                  T *__restrict__ filtered_all, int16_t *__restrict__ im_all,
                                                  int fme_level, int16_t *__restrict__ cols_all,
                                                  const int8_t *__restrict__ hpel_off)
{
  constexpr int shift1 = PixTraits<T>::bd - 8;
  const int b = blockIdx.x;
  const T *src = src_plane + src_off[b];
  T *filtered = filtered_all + (size_t)b * 4 * 4096;
  int16_t *im = im_all + (size_t)b * 5 * KVZ_CUDA_IPOL_IM_SIZE;
  int16_t *cols = cols_all + (size_t)b * 5 * KVZ_CUDA_IPOL_FIRST_COLS;
  const int hox = hpel_off ? hpel_off[2 * b] : 0, hoy = hpel_off ? hpel_off[2 * b + 1] : 0;
  const int rows = h + 7 + 1;
#define IM(k) (im + (k) * KVZ_CUDA_IPOL_IM_SIZE)
#define COL(k) (cols + (k) * KVZ_CUDA_IPOL_FIRST_COLS)
#define FLT(k) (filtered + (k) * 4096)
  if (stage == 0) {
    fme_hor<T>(src, ss, w, rows, 0, c_luma_fir[0], IM(0), COL(0));
    fme_hor<T>(src, ss, w, rows, fme_level > 1 ? 0 : 1, c_luma_fir[2], IM(1), COL(2));
    __syncthreads();
    for (int i = threadIdx.x; i < w * h; i += blockDim.x) {
      const int y = i / w, x = i - y * w;
      // right: horizontal half-pel; left: the same shifted by one column, column 0 from the first-column array
      FLT(1)[y * 64 + x] = (T)fme_round<T>(IM(1)[(y + 4) * 64 + x]);
      FLT(0)[y * 64 + x] = (T)fme_round<T>(x == 0 ? COL(2)[y + 4] : IM(1)[(y + 4) * 64 + x - 1]);
    }
    for (int i = threadIdx.x; i < w * (h + 1); i += blockDim.x) {
      const int y = i / w, x = i - y * w;   // vertical half-pel at rows y (top) = rows y-1 of bottom
      const int16_t s = (int16_t)(fir8_px<T>(c_luma_fir[2], src + (long)(y - 3) * ss + x + 1, ss) >> shift1);
      const T v = (T)fme_round<T>(s);
      if (y < h) FLT(2)[y * 64 + x] = v;
      if (y > 0) FLT(3)[(y - 1) * 64 + x] = v;
    }
  } else if (stage == 1) {
    for (int i = threadIdx.x; i < (w + 1) * (h + 1); i += blockDim.x) {
      const int y = i / (w + 1), x = i % (w + 1) - 1;      // x = -1: column from the first-column array
      const int16_t s = x < 0 ? (int16_t)(fir8_im(c_luma_fir[2], COL(2) + y, 1) >> 6)
                              : (int16_t)(fir8_im(c_luma_fir[2], IM(1) + y * 64 + x, 64) >> 6);
      const T v = (T)fme_round<T>(s);
      // v is the diagonal half-pel sample at (column x, row y) of the (w+1) x (h+1) lattice:
      //   top-right block uses (x, y), top-left (x+1 <- x), bottom-right (y-1), bottom-left both shifted.
      if (x >= 0 && y < h) FLT(1)[y * 64 + x] = v;
      if (x + 1 < w && y < h) FLT(0)[y * 64 + x + 1] = v;
      if (x >= 0 && y > 0) FLT(3)[(y - 1) * 64 + x] = v;
      if (x + 1 < w && y > 0) FLT(2)[(y - 1) * 64 + x + 1] = v;
    }
  } else {
    const int off_x_l = hox < 1 ? 0 : 1, off_x_r = hox < 0 ? 0 : 1;
    const int off_y_t = hoy < 1 ? 0 : 1, off_y_b = hoy < 0 ? 0 : 1;
    const int8_t *vt = hoy != 0 ? c_luma_fir[1] : c_luma_fir[3];
    const int8_t *vb = hoy != 0 ? c_luma_fir[3] : c_luma_fir[1];
    if (stage == 2) {
      const int8_t *hfl = hox != 0 ? c_luma_fir[1] : c_luma_fir[3];
      const int8_t *hfr = hox != 0 ? c_luma_fir[3] : c_luma_fir[1];
      fme_hor<T>(src, ss, w, rows, 0, hfl, IM(3), COL(1));
      fme_hor<T>(src, ss, w, rows, 0, hfr, IM(4), COL(3));
      __syncthreads();
      const int sample_off_y = hoy < 0 ? 0 : 1, sample_off_x = hox > -1 ? 1 : 0;
      const int8_t *vlr = hoy != 0 ? c_luma_fir[2] : c_luma_fir[0];
      const int16_t *hp_im = hox != 0 ? IM(1) : IM(0);
      const int16_t *hp_col = hox != 0 ? COL(2) : COL(0);
      fme_ver_plane<T>(FLT(0), w, h, vlr, IM(3), COL(1), !off_x_l, sample_off_y);
      fme_ver_plane<T>(FLT(1), w, h, vlr, IM(4), COL(3), !off_x_r, sample_off_y);
      fme_ver_plane<T>(FLT(2), w, h, vt, hp_im, hp_col, !sample_off_x, off_y_t);
      fme_ver_plane<T>(FLT(3), w, h, vb, hp_im, hp_col, !sample_off_x, off_y_b);
    } else {
      fme_ver_plane<T>(FLT(0), w, h, vt, IM(3), COL(1), !off_x_l, off_y_t);
      fme_ver_plane<T>(FLT(1), w, h, vt, IM(4), COL(3), !off_x_r, off_y_t);
      fme_ver_plane<T>(FLT(2), w, h, vb, IM(3), COL(1), !off_x_l, off_y_b);
      fme_ver_plane<T>(FLT(3), w, h, vb, IM(4), COL(3), !off_x_r, off_y_b);
    }
  }
#undef IM
#undef COL
#undef FLT
}

// get_extended_block's border-replicating copy (ref: ipol-generic.c:761-814)
template <class T>
__global__ void __launch_bounds__(256) extend_block_kernel(const T *__restrict__ src, int src_w, int src_h, int src_s,
                                                           int blk_x, int blk_y, int blk_w, int blk_h, int pad_l,
                                                           int pad_r, int pad_t, int pad_b, int pad_b_simd,
                                                           T *__restrict__ buf)
{
  const int es = pad_l + blk_w + pad_r, rows = pad_t + blk_h + pad_b;
  const int total = es * (rows + pad_b_simd) + 1;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int y = i / es, x = i - y * es;
    T v = 0;
    if (y < rows) {
      const int cy = clip3(0, src_h - 1, blk_y - pad_t + y), cx = clip3(0, src_w - 1, blk_x - pad_l + x);
      v = src[(long)cy * src_s + cx];
    }
    buf[i] = v;
  }
}

}  // namespace kvzc

using namespace kvzc;

extern "C" {

int kvz_cuda_sample_batch(int kind, int bitdepth, const void *src_plane, int src_stride, void *dst_base,
                          int dst_stride, const kvz_cuda_ipol *descs, int count, void *stream)
{
  KVZC_REQUIRE_DEVICE();
  KVZC_ARG(src_plane && dst_base && descs && kind >= 0 && kind <= 3);
  if (count == 0) return 0;
  if (bitdepth == 8) sample_kernel<uint8_t><<<count, 256, 0, as_stream(stream)>>>(kind, (const uint8_t *)src_plane, src_stride, dst_base, dst_stride, descs);
  else sample_kernel<uint16_t><<<count, 256, 0, as_stream(stream)>>>(kind, (const uint16_t *)src_plane, src_stride, dst_base, dst_stride, descs);
  KVZC_LAUNCHED();
  return 0;
}

int kvz_cuda_filter_fme_batch(int stage, int bitdepth, const void *src_plane, int src_stride, const int32_t *src_off,
                              int w, int h, void *filtered, int16_t *hor_intermediate, int fme_level,
                              int16_t *hor_first_cols, const int8_t *hpel_off, int count, void *stream)
{
  KVZC_REQUIRE_DEVICE();
  KVZC_ARG(src_plane && src_off && filtered && hor_intermediate && hor_first_cols && stage >= 0 && stage <= 3);
  KVZC_ARG(w >= 4 && w <= 64 && h >= 4 && h <= 64);
  if (count == 0) return 0;
  if (bitdepth == 8) fme_kernel<uint8_t><<<count, 256, 0, as_stream(stream)>>>(stage, (const uint8_t *)src_plane, src_stride, src_off, w, h, (uint8_t *)filtered, hor_intermediate, fme_level, hor_first_cols, hpel_off);
  else fme_kernel<uint16_t><<<count, 256, 0, as_stream(stream)>>>(stage, (const uint16_t *)src_plane, src_stride, src_off, w, h, (uint16_t *)filtered, hor_intermediate, fme_level, hor_first_cols, hpel_off);
  KVZC_LAUNCHED();
  return 0;
}

int kvz_cuda_extend_block(int bitdepth, const void *src, int src_w, int src_h, int src_s, int blk_x, int blk_y,
                          int blk_w, int blk_h, int pad_l, int pad_r, int pad_t, int pad_b, int pad_b_simd, void *buf,
                          void *stream)
{
  KVZC_REQUIRE_DEVICE();
  KVZC_ARG(src && buf && blk_w > 0 && blk_h > 0);
  const int total = (pad_l + blk_w + pad_r) * (pad_t + blk_h + pad_b + pad_b_simd) + 1;
  const int grid = (total + 255) / 256;
  if (bitdepth == 8) extend_block_kernel<uint8_t><<<grid, 256, 0, as_stream(stream)>>>((const uint8_t *)src, src_w, src_h, src_s, blk_x, blk_y, blk_w, blk_h, pad_l, pad_r, pad_t, pad_b, pad_b_simd, (uint8_t *)buf);
  else extend_block_kernel<uint16_t><<<grid, 256, 0, as_stream(stream)>>>((const uint16_t *)src, src_w, src_h, src_s, blk_x, blk_y, blk_w, blk_h, pad_l, pad_r, pad_t, pad_b, pad_b_simd, (uint16_t *)buf);
  KVZC_LAUNCHED();
  return 0;
}

}  // extern "C"
