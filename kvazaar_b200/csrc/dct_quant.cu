// dct_quant.cu -- dct group (DCT/IDCT 4..32, DST 4) and quant group (quant, dequant, quantize_residual,
// coeff_abs_sum, fast_coeff_cost).  Reference: src/strategies/generic/dct-generic.c, quant-generic.c.
#include "common.cuh"
#include "transform.cuh"

namespace kvzc {

// One CTA handles G = max(1, 256 / N^2) transform blocks; both passes run out of shared memory.
__global__ void __launch_bounds__(256) transform_kernel(int kind, int n, int bitdepth, const int16_t *__restrict__ in,
                                                        int16_t *__restrict__ out, int count, int g_per_cta)
{
  __shared__ int16_t s_a[32 * 32];
  __shared__ int16_t s_b[32 * 32];
  __shared__ int8_t s_m[32 * 32];
  const bool inverse = kind == KVZ_CUDA_TR_IDCT || kind == KVZ_CUDA_TR_IDST;
  const bool dst = kind == KVZ_CUDA_TR_DST || kind == KVZ_CUDA_TR_IDST;
  const int nn = n * n;
  const int first = blockIdx.x * g_per_cta;
  const int g = min(g_per_cta, count - first);
  load_matrix(s_m, n, dst, !inverse);
  const uint32_t *src32 = reinterpret_cast<const uint32_t *>(in + (size_t)first * nn);
  uint32_t *sa32 = reinterpret_cast<uint32_t *>(s_a);
  for (int e = threadIdx.x; e < g * nn / 2; e += blockDim.x) sa32[e] = __ldg(src32 + e);
  __syncthreads();
  const int l2 = ilog2(n);
  if (!inverse) {
    fwd_pass(s_a, s_b, s_m, n, g, l2 - 1 + (bitdepth - 8));   // ref: dct-generic.c:582-583
    __syncthreads();
    fwd_pass(s_b, s_a, s_m, n, g, l2 + 6);
  } else {
    inv_pass(s_a, s_b, s_m, n, g, 7);                          // ref: dct-generic.c:593-594
    __syncthreads();
    inv_pass(s_b, s_a, s_m, n, g, 12 - (bitdepth - 8));
  }
  __syncthreads();
  uint32_t *dst32 = reinterpret_cast<uint32_t *>(out + (size_t)first * nn);
  for (int e = threadIdx.x; e < g * nn / 2; e += blockDim.x) dst32[e] = sa32[e];
}

// quant / dequant of `count` n x n blocks, one CTA per block
__global__ void __launch_bounds__(256) quant_kernel(kvz_cuda_quant_params p, const int16_t *__restrict__ coef,
                                                    int16_t *__restrict__ q_coef, int n, int type,
                                                    const int8_t *__restrict__ scan_idx)
{
  __shared__ int16_t s_c[32 * 32];
  __shared__ int16_t s_q[32 * 32];
  __shared__ int32_t s_d[32 * 32];
  const int nn = n * n;
  const size_t base = (size_t)blockIdx.x * nn;
  for (int e = threadIdx.x; e < nn; e += blockDim.x) s_c[e] = coef[base + e];
  __syncthreads();
  quant_block(p, s_c, s_q, s_d, n, type, scan_idx ? scan_idx[blockIdx.x] : 0);
  __syncthreads();
  for (int e = threadIdx.x; e < nn; e += blockDim.x) q_coef[base + e] = s_q[e];
}

__global__ void __launch_bounds__(256) dequant_kernel(kvz_cuda_quant_params p, const int16_t *__restrict__ q_coef,
                                                      int16_t *__restrict__ coef, int n, int type, long total)
{
  const int transform_shift = 15 - p.bitdepth - ilog2(n);
  const int qp_scaled = scaled_qp(type, p.qp, (p.bitdepth - 8) * 6);
  const int shift = 20 - 14 - transform_shift;
  const int scale = c_inv_quant_scales[qp_scaled % 6] << (qp_scaled / 6);
  const int add = 1 << (shift - 1);
  for (long e = (long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long)gridDim.x * blockDim.x)
    coef[e] = (int16_t)clip3(-32768, 32767, ((int)q_coef[e] * scale + add) >> shift);
}

// kvz_quantize_residual, RDOQ-off branch (ref: quant-generic.c:198-292): one CTA per TU.
template <class T>
__global__ void __launch_bounds__(256) quantize_residual_kernel(kvz_cuda_quant_params p, const T *__restrict__ ref_plane,
                                                                const T *__restrict__ pred_plane, int in_stride,
                                                                T *__restrict__ rec_plane, int out_stride,
                                                                int16_t *__restrict__ coeff_out,
                                                                const kvz_cuda_tu *__restrict__ tus,
                                                                int32_t *__restrict__ has_coeffs, int phase_override)
{
  __shared__ TuScratch s;
  const kvz_cuda_tu tu = tus[blockIdx.x];
  const int has = quantize_residual_tu<T>(s, p, tu.width, tu.color, tu.scan_idx, tu.use_trskip, tu.cu_is_intra,
                                          tu.early_skip, phase_override >= 0 ? phase_override : tu.phase, ref_plane + tu.off_ref, in_stride,
                                          pred_plane + tu.off_pred, in_stride, rec_plane + tu.off_rec, out_stride,
                                          coeff_out + tu.off_coeff);
  if (threadIdx.x == 0) has_coeffs[blockIdx.x] = has;
}

// coeff_abs_sum (ref: quant-generic.c:342-349) / fast_coeff_cost (:351-375): one warp per array
__global__ void __launch_bounds__(128) coeff_sum_kernel(const int16_t *__restrict__ c, size_t length, int count,
                                                        int use_weights, unsigned long long weights,
                                                        uint32_t *__restrict__ out)
{
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= count) return;
  const int16_t *p = c + (size_t)warp * length;
  uint32_t s = 0;
  for (size_t i = lane; i < length; i += 32) {
    uint32_t a = (uint32_t)abs((int)p[i]);
    if (use_weights) { if (a > 3) a = 3; a = (uint32_t)((weights >> (16 * a)) & 0xffff); }
    s += a;
  }
  s = (uint32_t)warp_sum((int)s);
  if (lane == 0) out[warp] = s;
}

}  // namespace kvzc

using namespace kvzc;

extern "C" {

int kvz_cuda_transform_batch(int kind, int n, int bitdepth, const int16_t *in, int16_t *out, int count, void *stream)
{
  KVZC_REQUIRE_DEVICE();
  KVZC_ARG(in && out && count >= 0 && kind >= 0 && kind <= 3);
  KVZC_ARG(n == 4 || ((kind == KVZ_CUDA_TR_DCT || kind == KVZ_CUDA_TR_IDCT) && (n == 8 || n == 16 || n == 32)));
  if (count == 0) return 0;
  const int g = n * n >= 256 ? (n == 16 ? 4 : 1) : 1024 / (n * n);   // blocks per CTA (<= 1024 coefficients staged)
  transform_kernel<<<(count + g - 1) / g, 256, 0, as_stream(stream)>>>(kind, n, bitdepth, in, out, count, g);
  KVZC_LAUNCHED();
  return 0;
}

static int check_qp(const kvz_cuda_quant_params *p)
{
  KVZC_ARG(p != nullptr);
  if (p->scaling_list_enable) { set_error("scaling lists are not supported by the cuda strategy (flat lists only)"); return KVZ_CUDA_E_ARG; }
  KVZC_ARG(p->bitdepth >= 8 && p->bitdepth <= 10 && p->qp >= -12 && p->qp <= 63);
  return 0;
}

int kvz_cuda_quant_batch(const kvz_cuda_quant_params *p, const int16_t *coef, int16_t *q_coef, int n, int type,
                         const int8_t *scan_idx, int count, void *stream)
{
  KVZC_REQUIRE_DEVICE();
  if (int r = check_qp(p)) return r;
  KVZC_ARG(coef && q_coef && (n == 4 || n == 8 || n == 16 || n == 32));
  if (count == 0) return 0;
  quant_kernel<<<count, n * n < 256 ? (n * n < 32 ? 32 : n * n) : 256, 0, as_stream(stream)>>>(*p, coef, q_coef, n, type, scan_idx);
  KVZC_LAUNCHED();
  return 0;
}

int kvz_cuda_dequant_batch(const kvz_cuda_quant_params *p, const int16_t *q_coef, int16_t *coef, int n, int type,
                           int count, void *stream)
{
  KVZC_REQUIRE_DEVICE();
  if (int r = check_qp(p)) return r;
  KVZC_ARG(coef && q_coef && (n == 4 || n == 8 || n == 16 || n == 32));
  if (count == 0) return 0;
  const long total = (long)count * n * n;
  long gl = (total + 255) / 256; if (gl > (long)g_sm_count * 16) gl = (long)g_sm_count * 16;
  const int grid = (int)gl;
  dequant_kernel<<<grid, 256, 0, as_stream(stream)>>>(*p, q_coef, coef, n, type, total);
  KVZC_LAUNCHED();
  return 0;
}

int kvz_cuda_quantize_residual_batch(const kvz_cuda_quant_params *p, const void *ref_plane, const void *pred_plane,
                                     int in_stride, void *rec_plane, int out_stride, int16_t *coeff_out,
                                     const kvz_cuda_tu *tus, int count, int32_t *has_coeffs, void *stream)
{
  KVZC_REQUIRE_DEVICE();
  if (int r = check_qp(p)) return r;
  KVZC_ARG(ref_plane && pred_plane && rec_plane && coeff_out && tus && has_coeffs);
  if (count == 0) return 0;
  if (p->bitdepth == 8)
    quantize_residual_kernel<uint8_t><<<count, 256, 0, as_stream(stream)>>>(*p, (const uint8_t *)ref_plane, (const uint8_t *)pred_plane, in_stride, (uint8_t *)rec_plane, out_stride, coeff_out, tus, has_coeffs, -1);
  else
    quantize_residual_kernel<uint16_t><<<count, 256, 0, as_stream(stream)>>>(*p, (const uint16_t *)ref_plane, (const uint16_t *)pred_plane, in_stride, (uint16_t *)rec_plane, out_stride, coeff_out, tus, has_coeffs, -1);
  KVZC_LAUNCHED();
  return 0;
}

int kvz_cuda_quantize_residual_rdoq_batch(const kvz_cuda_quant_params *p, const kvz_cuda_rdoq_params *rp,
                                          const kvz_cuda_cabac_ctx *ctx_dev, const void *ref_plane, const void *pred_plane,
                                          int in_stride, void *rec_plane, int out_stride, int16_t *coeff_out,
                                          const kvz_cuda_tu *tus, int count, int widths_mask, int32_t *has_coeffs, void *stream)
{
  KVZC_REQUIRE_DEVICE();
  KVZC_ARG(p && rp && ctx_dev && ref_plane && pred_plane && rec_plane && coeff_out && tus && has_coeffs);
  KVZC_ARG(p->scaling_list_enable == 0 && (p->bitdepth == 8 || p->bitdepth == 10) && rp->bitdepth == p->bitdepth && rp->qp == p->qp);
  KVZC_ARG((widths_mask & ~(4 | 8 | 16 | 32)) == 0 && widths_mask != 0);
  if (count == 0) return 0;
  cudaStream_t st = as_stream(stream);
  for (int phase = 1; phase <= 2; ++phase) {
    if (p->bitdepth == 8)
      quantize_residual_kernel<uint8_t><<<count, 256, 0, st>>>(*p, (const uint8_t *)ref_plane, (const uint8_t *)pred_plane, in_stride, (uint8_t *)rec_plane, out_stride, coeff_out, tus, has_coeffs, phase);
    else
      quantize_residual_kernel<uint16_t><<<count, 256, 0, st>>>(*p, (const uint16_t *)ref_plane, (const uint16_t *)pred_plane, in_stride, (uint16_t *)rec_plane, out_stride, coeff_out, tus, has_coeffs, phase);
    KVZC_LAUNCHED();
    if (phase == 1)
      for (int n = 4; n <= 32; n <<= 1)
        if (widths_mask & n) if (int r = rdoq_launch_tus(*rp, ctx_dev, coeff_out, tus, count, n, st)) return r;
  }
  return 0;
}


int kvz_cuda_coeff_abs_sum_batch(const int16_t *coeffs, size_t length, int count, uint32_t *out, void *stream)
{
  KVZC_REQUIRE_DEVICE();
  KVZC_ARG(coeffs && out);
  if (count == 0) return 0;
  coeff_sum_kernel<<<(count * 32 + 127) / 128, 128, 0, as_stream(stream)>>>(coeffs, length, count, 0, 0ull, out);
  KVZC_LAUNCHED();
  return 0;
}

int kvz_cuda_fast_coeff_cost_batch(const int16_t *coeffs, int width, uint64_t weights, int count, uint32_t *out,
                                   void *stream)
{
  KVZC_REQUIRE_DEVICE();
  KVZC_ARG(coeffs && out && width > 0);
  if (count == 0) return 0;
  coeff_sum_kernel<<<(count * 32 + 127) / 128, 128, 0, as_stream(stream)>>>(coeffs, (size_t)width * width, count, 1, (unsigned long long)weights, out);
  KVZC_LAUNCHED();
  return 0;
}

}  // extern "C"
