// sao_nal.cu -- sao group (edge statistics, edge/band delta-distortion, reconstruction) and nal group (checksum).
// Reference: src/strategies/generic/sao-generic.c, sao_shared_generics.h, nal-generic.c; src/sao.c:180-202.
#include "common.cuh"

namespace kvzc {

// calc_sao_edge_dir for all four classes of one contiguous bw x bh block pair: one CTA per block.
template <class T>
__global__ void __launch_bounds__(256) sao_edge_stats_kernel(int bitdepth, const T *__restrict__ orig_base,
                                                             const T *__restrict__ rec_base,
                                                             const kvz_cuda_sao_blk *__restrict__ blks,
                                                             int32_t *__restrict__ out)
{
  __shared__ int s_acc[4][2][5];
  const kvz_cuda_sao_blk d = blks[blockIdx.x];
  const T *orig = orig_base + d.off_orig, *rec = rec_base + d.off_rec;
  const int bw = d.bw, bh = d.bh;
  const int so = d.stride_orig ? d.stride_orig : bw, sr = d.stride_rec ? d.stride_rec : bw;
  const int offset = bitdepth != 8 ? 1 << (bitdepth - 9) : 0, shift = bitdepth - 8;
  for (int i = threadIdx.x; i < 40; i += blockDim.x) (&s_acc[0][0][0])[i] = 0;
  __syncthreads();
  int sum[4][5], cnt[4][5];
#pragma unroll
  for (int e = 0; e < 4; ++e)
#pragma unroll
    for (int k = 0; k < 5; ++k) { sum[e][k] = 0; cnt[e][k] = 0; }
  const int iw = bw - 2, ih = bh - 2;
  for (int i = threadIdx.x; i < iw * ih; i += blockDim.x) {
    const int y = 1 + i / iw, x = 1 + i % iw;
    const int c = rec[y * sr + x];
    const int diff = ((int)orig[y * so + x] - c + offset) >> shift;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      int ax, ay;
      sao_eo_offsets(e, ax, ay);
      const int cat = sao_eo_cat(rec[(y + ay) * sr + x + ax], rec[(y - ay) * sr + x - ax], c);
#pragma unroll
      for (int k = 0; k < 5; ++k) { const int hit = cat == k; sum[e][k] += hit ? diff : 0; cnt[e][k] += hit; }
    }
  }
#pragma unroll
  for (int e = 0; e < 4; ++e)
#pragma unroll
    for (int k = 0; k < 5; ++k) {
      const int s = warp_sum(sum[e][k]), n = warp_sum(cnt[e][k]);
      if ((threadIdx.x & 31) == 0) { atomicAdd(&s_acc[e][0][k], s); atomicAdd(&s_acc[e][1][k], n); }
    }
  __syncthreads();
  for (int i = threadIdx.x; i < 40; i += blockDim.x) out[(size_t)blockIdx.x * 40 + i] = (&s_acc[0][0][0])[i];
}

template <class T>
__global__ void __launch_bounds__(256) sao_edge_dd_kernel(int bitdepth, const T *__restrict__ orig_base,
                                                          const T *__restrict__ rec_base,
                                                          const kvz_cuda_sao_blk *__restrict__ blks,
                                                          const int8_t *__restrict__ eo_class,
                                                          const int32_t *__restrict__ offsets, int32_t *__restrict__ out)
{
  const kvz_cuda_sao_blk d = blks[blockIdx.x];
  const T *orig = orig_base + d.off_orig, *rec = rec_base + d.off_rec;
  const int bw = d.bw, bh = d.bh, eo = eo_class[blockIdx.x];
  const int so = d.stride_orig ? d.stride_orig : bw, sr = d.stride_rec ? d.stride_rec : bw;
  const int bit_offset = bitdepth != 8 ? 1 << (bitdepth - 9) : 0, shift = bitdepth - 8;
  EdgeOffsets off;
#pragma unroll
  for (int k = 0; k < 5; ++k) off.o[k] = offsets[(size_t)blockIdx.x * 5 + k];
  int ax, ay;
  sao_eo_offsets(eo, ax, ay);
  int sum = 0;
  const int iw = bw - 2, ih = bh - 2;
  for (int i = threadIdx.x; i < iw * ih; i += blockDim.x) {
    const int y = 1 + i / iw, x = 1 + i % iw;
    const int c = rec[y * sr + x];
    const int cat = sao_eo_cat(rec[(y + ay) * sr + x + ax], rec[(y - ay) * sr + x - ax], c);
    const int o = off[cat];
    if (o != 0) {
      const int diff = ((int)orig[y * so + x] - c + bit_offset) >> shift;
      const int delta = diff - o;
      sum += delta * delta - diff * diff;
    }
  }
  sum = block_sum(sum);
  if (threadIdx.x == 0) out[blockIdx.x] = sum;
}

template <class T>
__global__ void __launch_bounds__(256) sao_band_dd_kernel(int bitdepth, const T *__restrict__ orig_base,
                                                          const T *__restrict__ rec_base,
                                                          const kvz_cuda_sao_blk *__restrict__ blks,
                                                          const int32_t *__restrict__ band_pos,
                                                          const int32_t *__restrict__ bands, int32_t *__restrict__ out)
{
  const kvz_cuda_sao_blk d = blks[blockIdx.x];
  const T *orig = orig_base + d.off_orig, *rec = rec_base + d.off_rec;
  const int shift = bitdepth - 5, bp = band_pos[blockIdx.x];
  const int so = d.stride_orig ? d.stride_orig : d.bw, sr = d.stride_rec ? d.stride_rec : d.bw;
  int bnd[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) bnd[k] = bands[(size_t)blockIdx.x * 4 + k];
  int sum = 0;
  for (int i = threadIdx.x; i < d.bw * d.bh; i += blockDim.x) {
    const int y = i / d.bw, x = i - y * d.bw;
    const int r = rec[y * sr + x];
    const int band = (r >> shift) - bp;
    int o = 0;
#pragma unroll
    for (int k = 0; k < 4; ++k) o = band == k ? bnd[k] : o;
    if (o != 0) {
      const int diff = (int)orig[y * so + x] - r;
      const int delta = diff - o;
      sum += delta * delta - diff * diff;
    }
  }
  sum = block_sum(sum);
  if (threadIdx.x == 0) out[blockIdx.x] = sum;
}

// sao_reconstruct_color (ref: sao-generic.c:84-124) with the band LUT of kvz_calc_sao_offset_array (sao.c:180-202)
// evaluated per sample.
template <class T>
__global__ void __launch_bounds__(256) sao_reconstruct_kernel(int bitdepth, const T *__restrict__ rec_base, int stride,
                                                              T *__restrict__ new_base, int new_stride,
                                                              const kvz_cuda_sao_rec *__restrict__ descs)
{
  const kvz_cuda_sao_rec d = descs[blockIdx.x];
  const T *rec = rec_base + d.off_rec;
  T *dst = new_base + d.off_new;
  const int offset_v = d.color == 2 ? 5 : 0;
  const int bp = d.band_position[d.color == 2 ? 1 : 0];
  int ax, ay;
  sao_eo_offsets(d.eo_class, ax, ay);
  for (int i = threadIdx.x; i < d.bw * d.bh; i += blockDim.x) {
    const int y = i / d.bw, x = i - y * d.bw;
    const T *c = rec + (long)y * stride + x;
    int v = c[0];
    if (d.type == 1) v = sao_band_px(v, bitdepth, bp, d.offsets + offset_v);
    else if (d.type == 2) v = sao_edge_px(v, c[ay * stride + ax], c[-ay * stride - ax], PixTraits<T>::bd, d.offsets + offset_v);
    dst[(long)y * new_stride + x] = (T)v;
  }
}

// HEVC picture checksum (ref: nal-generic.c:57-82): sum over pixels of (byte ^ mask(x,y)), both bytes for >8 bit.
// scratch[0] = running sum, scratch[1] = CTAs done; the last CTA writes the big-endian result.
template <class T>
__global__ void __launch_bounds__(256) checksum_kernel(const T *__restrict__ data, int height, int width, int stride,
                                                       uint32_t *__restrict__ scratch, uint8_t *__restrict__ out4)
{
  uint32_t s = 0;
  const long total = (long)height * width;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int y = (int)(i / width), x = (int)(i - (long)y * width);
    const uint32_t mask = (uint32_t)((x & 0xff) ^ (y & 0xff) ^ (x >> 8) ^ (y >> 8)) & 0xff;
    const uint32_t v = data[(long)y * stride + x];
    s += (v & 0xff) ^ mask;
    if (sizeof(T) == 2) s += ((v >> 8) & 0xff) ^ mask;
  }
  s = (uint32_t)block_sum((int)s);
  __shared__ bool s_last;
  if (threadIdx.x == 0) {
    atomicAdd(&scratch[0], s);
    __threadfence();
    s_last = atomicAdd(&scratch[1], 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (s_last && threadIdx.x == 0) {
    const uint32_t t = atomicAdd(&scratch[0], 0u);
    out4[0] = (uint8_t)(t >> 24); out4[1] = (uint8_t)(t >> 16); out4[2] = (uint8_t)(t >> 8); out4[3] = (uint8_t)t;
  }
}

}  // namespace kvzc

using namespace kvzc;

extern "C" {

int kvz_cuda_sao_edge_stats_batch(int bitdepth, const void *orig, const void *rec, const kvz_cuda_sao_blk *blks,
                                  int count, int32_t *cat_sum_cnt, void *stream)
{
  KVZC_REQUIRE_DEVICE();
  KVZC_ARG(orig && rec && blks && cat_sum_cnt);
  if (count == 0) return 0;
  if (bitdepth == 8) sao_edge_stats_kernel<uint8_t><<<count, 256, 0, as_stream(stream)>>>(bitdepth, (const uint8_t *)orig, (const uint8_t *)rec, blks, cat_sum_cnt);
  else sao_edge_stats_kernel<uint16_t><<<count, 256, 0, as_stream(stream)>>>(bitdepth, (const uint16_t *)orig, (const uint16_t *)rec, blks, cat_sum_cnt);
  KVZC_LAUNCHED();
  return 0;
}

int kvz_cuda_sao_edge_ddistortion_batch(int bitdepth, const void *orig, const void *rec, const kvz_cuda_sao_blk *blks,
                                        const int8_t *eo_class, const int32_t *offsets, int count, int32_t *out,
                                        void *stream)
{
  KVZC_REQUIRE_DEVICE();
  KVZC_ARG(orig && rec && blks && eo_class && offsets && out);
  if (count == 0) return 0;
  if (bitdepth == 8) sao_edge_dd_kernel<uint8_t><<<count, 256, 0, as_stream(stream)>>>(bitdepth, (const uint8_t *)orig, (const uint8_t *)rec, blks, eo_class, offsets, out);
  else sao_edge_dd_kernel<uint16_t><<<count, 256, 0, as_stream(stream)>>>(bitdepth, (const uint16_t *)orig, (const uint16_t *)rec, blks, eo_class, offsets, out);
  KVZC_LAUNCHED();
  return 0;
}

int kvz_cuda_sao_band_ddistortion_batch(int bitdepth, const void *orig, const void *rec, const kvz_cuda_sao_blk *blks,
                                        const int32_t *band_pos, const int32_t *bands, int count, int32_t *out,
                                        void *stream)
{
  KVZC_REQUIRE_DEVICE();
  KVZC_ARG(orig && rec && blks && band_pos && bands && out);
  if (count == 0) return 0;
  if (bitdepth == 8) sao_band_dd_kernel<uint8_t><<<count, 256, 0, as_stream(stream)>>>(bitdepth, (const uint8_t *)orig, (const uint8_t *)rec, blks, band_pos, bands, out);
  else sao_band_dd_kernel<uint16_t><<<count, 256, 0, as_stream(stream)>>>(bitdepth, (const uint16_t *)orig, (const uint16_t *)rec, blks, band_pos, bands, out);
  KVZC_LAUNCHED();
  return 0;
}

int kvz_cuda_sao_reconstruct_batch(int bitdepth, const void *rec, int stride, void *new_rec, int new_stride,
                                   const kvz_cuda_sao_rec *descs, int count, void *stream)
{
  KVZC_REQUIRE_DEVICE();
  KVZC_ARG(rec && new_rec && descs);
  if (count == 0) return 0;
  if (bitdepth == 8) sao_reconstruct_kernel<uint8_t><<<count, 256, 0, as_stream(stream)>>>(bitdepth, (const uint8_t *)rec, stride, (uint8_t *)new_rec, new_stride, descs);
  else sao_reconstruct_kernel<uint16_t><<<count, 256, 0, as_stream(stream)>>>(bitdepth, (const uint16_t *)rec, stride, (uint16_t *)new_rec, new_stride, descs);
  KVZC_LAUNCHED();
  return 0;
}

int kvz_cuda_array_checksum(int bitdepth, const void *data, int height, int width, int stride, uint8_t *out4,
                            void *stream)
{
  KVZC_REQUIRE_DEVICE();
  KVZC_ARG(data && out4 && height > 0 && width > 0);
  cudaStream_t st = as_stream(stream);
  uint32_t *scratch = nullptr;
  KVZC_CHECK(cudaMallocAsync((void **)&scratch, 8, st));
  KVZC_CHECK(cudaMemsetAsync(scratch, 0, 8, st));
  const long total = (long)height * width;
  long g = (total + 256 * 16 - 1) / (256 * 16);
  const int grid = (int)(g < 1 ? 1 : (g > g_sm_count * 8 ? g_sm_count * 8 : g));
  if (bitdepth == 8) checksum_kernel<uint8_t><<<grid, 256, 0, st>>>((const uint8_t *)data, height, width, stride, scratch, out4);
  else checksum_kernel<uint16_t><<<grid, 256, 0, st>>>((const uint16_t *)data, height, width, stride, scratch, out4);
  KVZC_LAUNCHED();
  KVZC_CHECK(cudaFreeAsync(scratch, st));
  return 0;
}

}  // extern "C"
