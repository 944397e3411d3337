// picture.cu -- picture-group kernels: SAD / SATD / SSD families, bipred average, pixel variance.
// Reference behaviour: src/strategies/generic/picture-generic.c, strategies-picture.h:53-113.
#include "common.cuh"
#include "satd.cuh"

namespace kvzc {

// ---------------------------------------------------------------------------------------------
// Contiguous NxN pairs.  Pair p: a at a_base + (p / M) * block_pitch + (p % M) * mode_pitch, b at (p / M) * N*N.
// (M = 1, block_pitch = N*N for the plain batch; M = num_modes for the *_dual / multi variants.)
// L = min(S*S, 32) lanes cooperate on one pair (S = N/8 sub-blocks per row), each lane owning whole 8x8
// sub-blocks; partial sums are combined with warp shuffles ("warp-shuffle Hadamard reductions").
// ---------------------------------------------------------------------------------------------
template <class T, int N>
__global__ void __launch_bounds__(128) satd_nxn_kernel(const T *__restrict__ a, const T *__restrict__ b,
                                                       long block_pitch, int mode_pitch, int M, int count_pairs,
                                                       uint32_t *__restrict__ out)
{
  constexpr int S = N / 8;
  constexpr int SUBS = S * S;
  constexpr int L = SUBS < 32 ? SUBS : 32;
  constexpr int SHIFT = PixTraits<T>::bd - 8;
  const long tid = (long)blockIdx.x * blockDim.x + threadIdx.x;
  const long pair = tid / L;
  const int lane = (int)(tid % L);
  uint32_t sum = 0;
  if (pair < count_pairs) {
    const T *pa = a + (pair / M) * block_pitch + (long)(pair % M) * mode_pitch;
    const T *pb = b + (pair / M) * (long)(N * N);
#pragma unroll 1
    for (int s = lane; s < SUBS; s += L) {
      const int sy = s / S, sx = s % S;
      const T *qa = pa + (sy * 8) * N + sx * 8;
      const T *qb = pb + (sy * 8) * N + sx * 8;
      if constexpr (sizeof(T) == 1) {
        uint2 ra[8], rb[8];
        if constexpr (N == 8) {   // 64 contiguous bytes: four 128-bit loads per operand
          const uint4 *va = reinterpret_cast<const uint4 *>(qa), *vb = reinterpret_cast<const uint4 *>(qb);
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const uint4 x = __ldg(va + j), y = __ldg(vb + j);
            ra[2 * j] = make_uint2(x.x, x.y); ra[2 * j + 1] = make_uint2(x.z, x.w);
            rb[2 * j] = make_uint2(y.x, y.y); rb[2 * j + 1] = make_uint2(y.z, y.w);
          }
        } else {
#pragma unroll
          for (int r = 0; r < 8; ++r) {
            ra[r] = __ldg(reinterpret_cast<const uint2 *>(qa + r * N));
            rb[r] = __ldg(reinterpret_cast<const uint2 *>(qb + r * N));
          }
        }
        sum += (hadamard8x8_u8(ra, rb) + 2) >> 2;
      } else {
        sum += satd_sub_strided<T, 8>(qa, N, qb, N);
      }
    }
  }
#pragma unroll
  for (int o = L / 2; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  if (pair < count_pairs && lane == 0) out[pair] = sum >> SHIFT;
}

// 4x4: one thread per pair, 16 contiguous bytes per operand (no bit-depth shift, ref: picture-generic.c:213-221).
template <class T>
__global__ void __launch_bounds__(256) satd_4x4_kernel(const T *__restrict__ a, const T *__restrict__ b,
                                                       long block_pitch, int mode_pitch, int M, int count_pairs,
                                                       uint32_t *__restrict__ out)
{
  const long pair = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (pair >= count_pairs) return;
  const T *pa = a + (pair / M) * block_pitch + (long)(pair % M) * mode_pitch;
  const T *pb = b + (pair / M) * 16L;
  if constexpr (sizeof(T) == 1) {
    const uint4 x = __ldg(reinterpret_cast<const uint4 *>(pa)), y = __ldg(reinterpret_cast<const uint4 *>(pb));
    const uint32_t ra[4] = { x.x, x.y, x.z, x.w }, rb[4] = { y.x, y.y, y.z, y.w };
    out[pair] = (hadamard4x4_u8(ra, rb) + 1) >> 1;
  } else {
    out[pair] = satd_sub_strided<T, 4>(pa, 4, pb, 4);
  }
}

// SAD of contiguous NxN pairs: 16-byte chunks, L lanes per pair, shuffle reduce.
template <class T, int N>
__global__ void __launch_bounds__(128) sad_nxn_kernel(const T *__restrict__ a, const T *__restrict__ b,
                                                      long block_pitch, int mode_pitch, int M, int count_pairs,
                                                      uint32_t *__restrict__ out)
{
  constexpr int CHUNKS = N * N * (int)sizeof(T) / 16;
  constexpr int L = CHUNKS < 32 ? CHUNKS : 32;
  constexpr int SHIFT = PixTraits<T>::bd - 8;
  const long tid = (long)blockIdx.x * blockDim.x + threadIdx.x;
  const long pair = tid / L;
  const int lane = (int)(tid % L);
  uint32_t sum = 0;
  if (pair < count_pairs) {
    const uint4 *va = reinterpret_cast<const uint4 *>(a + (pair / M) * block_pitch + (long)(pair % M) * mode_pitch);
    const uint4 *vb = reinterpret_cast<const uint4 *>(b + (pair / M) * (long)(N * N));
    for (int c = lane; c < CHUNKS; c += L) {
      const uint4 x = __ldg(va + c), y = __ldg(vb + c);
      if constexpr (sizeof(T) == 1) {
        sum = __dp4a(__vabsdiffu4(x.x, y.x), 0x01010101u, sum);
        sum = __dp4a(__vabsdiffu4(x.y, y.y), 0x01010101u, sum);
        sum = __dp4a(__vabsdiffu4(x.z, y.z), 0x01010101u, sum);
        sum = __dp4a(__vabsdiffu4(x.w, y.w), 0x01010101u, sum);
      } else {
        const uint32_t xs[4] = { x.x, x.y, x.z, x.w }, ys[4] = { y.x, y.y, y.z, y.w };
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          sum += (uint32_t)abs((int)(xs[k] & 0xffff) - (int)(ys[k] & 0xffff));
          sum += (uint32_t)abs((int)(xs[k] >> 16) - (int)(ys[k] >> 16));
        }
      }
    }
  }
#pragma unroll
  for (int o = L / 2; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  if (pair < count_pairs && lane == 0) out[pair] = sum >> SHIFT;
}

template <class T, bool SATD>
static int launch_nxn(int n, const T *a, const T *b, long block_pitch, int mode_pitch, int M, int pairs, uint32_t *out,
                      cudaStream_t st)
{
  if (pairs == 0) return 0;
#define KVZC_GO(KERN, NN, LANES, TPB)                                                             \
  {                                                                                               \
    const long threads = (long)pairs * (LANES);                                                   \
    const int grid = (int)((threads + (TPB) - 1) / (TPB));                                        \
    KERN<<<grid, (TPB), 0, st>>>(a, b, block_pitch, mode_pitch, M, pairs, out);                   \
    KVZC_LAUNCHED();                                                                              \
    return 0;                                                                                     \
  }
  if constexpr (SATD) {
    switch (n) {
      case 4: KVZC_GO(satd_4x4_kernel<T>, 4, 1, 256)
      case 8: KVZC_GO((satd_nxn_kernel<T, 8>), 8, 1, 128)
      case 16: KVZC_GO((satd_nxn_kernel<T, 16>), 16, 4, 128)
      case 32: KVZC_GO((satd_nxn_kernel<T, 32>), 32, 16, 128)
      case 64: KVZC_GO((satd_nxn_kernel<T, 64>), 64, 32, 128)
    }
  } else {
    constexpr int PB = 16 / (int)sizeof(T);   // pixels per 16-byte chunk
    switch (n) {
      case 4: KVZC_GO((sad_nxn_kernel<T, 4>), 4, (16 / PB < 32 ? 16 / PB : 32), 128)
      case 8: KVZC_GO((sad_nxn_kernel<T, 8>), 8, (64 / PB < 32 ? 64 / PB : 32), 128)
      case 16: KVZC_GO((sad_nxn_kernel<T, 16>), 16, (256 / PB < 32 ? 256 / PB : 32), 128)
      case 32: KVZC_GO((sad_nxn_kernel<T, 32>), 32, 32, 128)
      case 64: KVZC_GO((sad_nxn_kernel<T, 64>), 64, 32, 128)
    }
  }
#undef KVZC_GO
  set_error("unsupported block size %d", n);
  return KVZ_CUDA_E_ARG;
}

// ---------------------------------------------------------------------------------------------
// Strided block costs: one warp per descriptor.
// ---------------------------------------------------------------------------------------------
template <class T>
__global__ void __launch_bounds__(128) block_cost_kernel(int op, const T *__restrict__ pa, int sa,
                                                         const T *__restrict__ pb, int sb,
                                                         const kvz_cuda_blk *__restrict__ descs, int count,
                                                         uint32_t *__restrict__ out)
{
  constexpr int SHIFT = PixTraits<T>::bd - 8;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= count) return;
  const kvz_cuda_blk d = descs[warp];
  const T *a = pa + d.off_a;
  const T *b = pb + d.off_b;
  int w = d.w, h = d.h;
  uint32_t sum = 0;
  if (op == KVZ_CUDA_OP_REG_SAD) {
    for (int i = lane; i < w * h; i += 32) { const int y = i / w, x = i - y * w; sum += abs((int)a[y * sa + x] - (int)b[y * sb + x]); }
  } else if (op == KVZ_CUDA_OP_SSD) {
    for (int i = lane; i < w * w; i += 32) { const int y = i / w, x = i - y * w; const int t = (int)a[y * sa + x] - (int)b[y * sb + x]; sum += t * t; }
  } else if (op == KVZ_CUDA_OP_VER_SAD) {
    for (int i = lane; i < w * h; i += 32) { const int y = i / w, x = i - y * w; sum += abs((int)a[y * sa + x] - (int)b[x]); }
  } else if (op == KVZ_CUDA_OP_HOR_SAD) {
    // ref: picture-generic.c:714-752.  Columns outside [left, w-right) compare against the replicated edge column.
    const int left = d.left, right = d.right;
    for (int i = lane; i < w * h; i += 32) {
      const int y = i / w, x = i - y * w;
      int rx = x;
      if (left) rx = max(x, left);
      else if (right) rx = min(x, w - right - 1);
      sum += abs((int)a[y * sa + x] - (int)b[y * sb + rx]);
    }
  } else {  // KVZ_CUDA_OP_SATD_ANY, ref: strategies-picture.h:75-113
    // enumerate the 4x4 column strip, the 4x4 row strip and the 8x8 interior as one list of sub-blocks
    const int wmod = w & 7, hmod = h & 7;
    const int n_col = wmod ? h / 4 : 0;
    const int w2 = w - (wmod ? 4 : 0), x0 = wmod ? 4 : 0;
    const int n_row = hmod ? w2 / 4 : 0;
    const int h2 = h - (hmod ? 4 : 0), y0 = hmod ? 4 : 0;
    const int n8x = w2 / 8, n8 = n8x * (h2 / 8);
    for (int i = lane; i < n_col + n_row + n8; i += 32) {
      if (i < n_col) sum += satd4_sub<T>(a + (i * 4) * sa, sa, b + (i * 4) * sb, sb);
      else if (i < n_col + n_row) { const int x = x0 + (i - n_col) * 4; sum += satd4_sub<T>(a + x, sa, b + x, sb); }
      else {
        const int j = i - n_col - n_row, by = y0 + (j / n8x) * 8, bx = x0 + (j % n8x) * 8;
        sum += satd8_sub<T>(a + by * sa + bx, sa, b + by * sb + bx, sb);
      }
    }
  }
  sum = (uint32_t)warp_sum((int)sum);
  if (lane == 0) {
    if (op == KVZ_CUDA_OP_SATD_ANY) sum >>= SHIFT;
    else if (op == KVZ_CUDA_OP_SSD) sum = (uint32_t)((int)sum >> (2 * SHIFT));
    out[warp] = sum;
  }
}

// satd_any_size_quad: one warp per descriptor, 4 predictions against one original.
// Reproduces ref: picture-generic.c:404-471 literally, including that for height % 8 == 4 the 8x8 pass restarts
// at row 0 (rows 0..3 are counted twice, the last four rows never) and that the 4x4 row strip starts at column 0.
template <class T>
__global__ void __launch_bounds__(128) satd_quad_kernel(const T *__restrict__ pred_base, int ps,
                                                        const T *__restrict__ orig_base, int os,
                                                        const kvz_cuda_quad *__restrict__ descs, int count,
                                                        uint32_t *__restrict__ costs)
{
  constexpr int SHIFT = PixTraits<T>::bd - 8;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= count) return;
  const kvz_cuda_quad d = descs[warp];
  const T *orig = orig_base + d.off_orig;
  int w = d.w, h = d.h;
  const int wmod = w & 7;
  const int n_col = wmod ? h / 4 : 0;
  if (wmod) w -= 4;
  const int n_row = (h & 7) ? w / 4 : 0;
  if (h & 7) h -= 4;
  const int n8x = (w - wmod + 7) / 8;               // x = wmod, wmod+8, ... < w
  const int n8 = n8x * (h / 8);
  uint32_t sum[4] = { 0, 0, 0, 0 };
  for (int i = lane; i < n_col + n_row + n8; i += 32) {
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const T *p = pred_base + d.off_pred[k];
      if (i < n_col) sum[k] += satd4_sub<T>(orig + (i * 4) * os, os, p + (i * 4) * ps, ps);
      else if (i < n_col + n_row) { const int x = (i - n_col) * 4; sum[k] += satd4_sub<T>(orig + x, os, p + x, ps); }
      else {
        const int j = i - n_col - n_row, by = (j / n8x) * 8, bx = wmod + (j % n8x) * 8;
        sum[k] += satd8_sub<T>(orig + by * os + bx, os, p + by * ps + bx, ps);
      }
    }
  }
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const uint32_t s = (uint32_t)warp_sum((int)sum[k]);
    if (lane == 0) costs[warp * 4 + k] = s >> SHIFT;
  }
}

// bipred average of one plane, ref: picture-generic.c:553-632
template <class T>
__global__ void bipred_plane_kernel(T *__restrict__ dst, int dst_stride, const void *__restrict__ l0,
                                    const void *__restrict__ l1, int im0, int im1, int w, int h)
{
  constexpr int BITS = PixTraits<T>::bd;
  const int shift = 15 - BITS, offset = 1 << (shift - 1);
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= w * h) return;
  const int16_t s0 = im0 ? ((const int16_t *)l0)[i] : (int16_t)(((const T *)l0)[i] << (14 - BITS));
  const int16_t s1 = im1 ? ((const int16_t *)l1)[i] : (int16_t)(((const T *)l1)[i] << (14 - BITS));
  const int r = ((int)s0 + (int)s1 + offset) >> shift;
  dst[(i / w) * dst_stride + (i % w)] = (T)clip3(0, (1 << BITS) - 1, r);
}

// pixel_var: double accumulation order is part of the result -> one thread per array, sequential
// (ref: picture-generic.c:755-778).  -fmad=false keeps tmp*tmp and the add separate like the C code.
template <class T>
__global__ void pixel_var_kernel(const T *__restrict__ buf, uint32_t len, int count, double *__restrict__ out)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  const T *p = buf + (size_t)i * len;
  double sum = 0;
  for (uint32_t k = 0; k < len; ++k) sum += p[k];
  const double mean = sum / (double)len;
  double var = 0;
  for (uint32_t k = 0; k < len; ++k) { const double t = (double)p[k] - mean; var = __dadd_rn(var, __dmul_rn(t, t)); }
  out[i] = var / len;
}

}  // namespace kvzc

using namespace kvzc;

extern "C" {

int kvz_cuda_sad_nxn_batch(int n, int bitdepth, const void *a, const void *b, int count, uint32_t *out, void *stream)
{
  KVZC_REQUIRE_DEVICE();
  KVZC_ARG(a && b && out && count >= 0);
  if (bitdepth == 8) return launch_nxn<uint8_t, false>(n, (const uint8_t *)a, (const uint8_t *)b, n * n, 0, 1, count, out, as_stream(stream));
  return launch_nxn<uint16_t, false>(n, (const uint16_t *)a, (const uint16_t *)b, n * n, 0, 1, count, out, as_stream(stream));
}

int kvz_cuda_satd_nxn_batch(int n, int bitdepth, const void *a, const void *b, int count, uint32_t *out, void *stream)
{
  KVZC_REQUIRE_DEVICE();
  KVZC_ARG(a && b && out && count >= 0);
  if (bitdepth == 8) return launch_nxn<uint8_t, true>(n, (const uint8_t *)a, (const uint8_t *)b, n * n, 0, 1, count, out, as_stream(stream));
  return launch_nxn<uint16_t, true>(n, (const uint16_t *)a, (const uint16_t *)b, n * n, 0, 1, count, out, as_stream(stream));
}

int kvz_cuda_cost_nxn_multi_batch(int use_satd, int n, int bitdepth, const void *preds, int64_t block_pitch,
                                  int mode_pitch, int num_modes, const void *orig, int count, uint32_t *costs,
                                  void *stream)
{
  KVZC_REQUIRE_DEVICE();
  KVZC_ARG(preds && orig && costs && count >= 0 && num_modes >= 1);
  const int pairs = count * num_modes;
  cudaStream_t st = as_stream(stream);
  if (bitdepth == 8) {
    KVZC_ARG((block_pitch % 16) == 0 && (mode_pitch % 16) == 0);
    return use_satd ? launch_nxn<uint8_t, true>(n, (const uint8_t *)preds, (const uint8_t *)orig, block_pitch, mode_pitch, num_modes, pairs, costs, st)
                    : launch_nxn<uint8_t, false>(n, (const uint8_t *)preds, (const uint8_t *)orig, block_pitch, mode_pitch, num_modes, pairs, costs, st);
  }
  KVZC_ARG((block_pitch % 8) == 0 && (mode_pitch % 8) == 0);
  return use_satd ? launch_nxn<uint16_t, true>(n, (const uint16_t *)preds, (const uint16_t *)orig, block_pitch, mode_pitch, num_modes, pairs, costs, st)
                  : launch_nxn<uint16_t, false>(n, (const uint16_t *)preds, (const uint16_t *)orig, block_pitch, mode_pitch, num_modes, pairs, costs, st);
}

int kvz_cuda_block_cost_batch(int op, int bitdepth, const void *plane_a, int stride_a, const void *plane_b,
                              int stride_b, const kvz_cuda_blk *descs, int count, uint32_t *out, void *stream)
{
  KVZC_REQUIRE_DEVICE();
  KVZC_ARG(plane_a && plane_b && descs && out && op >= 0 && op <= KVZ_CUDA_OP_HOR_SAD);
  if (count == 0) return 0;
  const int grid = (count * 32 + 127) / 128;
  if (bitdepth == 8)
    block_cost_kernel<uint8_t><<<grid, 128, 0, as_stream(stream)>>>(op, (const uint8_t *)plane_a, stride_a, (const uint8_t *)plane_b, stride_b, descs, count, out);
  else
    block_cost_kernel<uint16_t><<<grid, 128, 0, as_stream(stream)>>>(op, (const uint16_t *)plane_a, stride_a, (const uint16_t *)plane_b, stride_b, descs, count, out);
  KVZC_LAUNCHED();
  return 0;
}

int kvz_cuda_satd_any_size_quad_batch(int bitdepth, const void *pred_base, int pred_stride, const void *orig_base,
                                      int orig_stride, const kvz_cuda_quad *descs, int count, uint32_t *costs,
                                      void *stream)
{
  KVZC_REQUIRE_DEVICE();
  KVZC_ARG(pred_base && orig_base && descs && costs);
  if (count == 0) return 0;
  const int grid = (count * 32 + 127) / 128;
  if (bitdepth == 8)
    satd_quad_kernel<uint8_t><<<grid, 128, 0, as_stream(stream)>>>((const uint8_t *)pred_base, pred_stride, (const uint8_t *)orig_base, orig_stride, descs, count, costs);
  else
    satd_quad_kernel<uint16_t><<<grid, 128, 0, as_stream(stream)>>>((const uint16_t *)pred_base, pred_stride, (const uint16_t *)orig_base, orig_stride, descs, count, costs);
  KVZC_LAUNCHED();
  return 0;
}

int kvz_cuda_bipred_average_plane(int bitdepth, void *dst, int dst_stride, const void *l0, const void *l1,
                                  int l0_is_im, int l1_is_im, int w, int h, void *stream)
{
  KVZC_REQUIRE_DEVICE();
  KVZC_ARG(dst && l0 && l1 && w > 0 && h > 0);
  const int grid = (w * h + 255) / 256;
  if (bitdepth == 8) bipred_plane_kernel<uint8_t><<<grid, 256, 0, as_stream(stream)>>>((uint8_t *)dst, dst_stride, l0, l1, l0_is_im, l1_is_im, w, h);
  else bipred_plane_kernel<uint16_t><<<grid, 256, 0, as_stream(stream)>>>((uint16_t *)dst, dst_stride, l0, l1, l0_is_im, l1_is_im, w, h);
  KVZC_LAUNCHED();
  return 0;
}

int kvz_cuda_pixel_var_batch(int bitdepth, const void *buf, uint32_t len, int count, double *out, void *stream)
{
  KVZC_REQUIRE_DEVICE();
  KVZC_ARG(buf && out && len > 0);
  if (count == 0) return 0;
  const int grid = (count + 63) / 64;
  if (bitdepth == 8) pixel_var_kernel<uint8_t><<<grid, 64, 0, as_stream(stream)>>>((const uint8_t *)buf, len, count, out);
  else pixel_var_kernel<uint16_t><<<grid, 64, 0, as_stream(stream)>>>((const uint16_t *)buf, len, count, out);
  KVZC_LAUNCHED();
  return 0;
}

}  // extern "C"
