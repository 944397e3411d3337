// transform.cuh -- block-cooperative HEVC integer transforms and (de)quantisation on shared memory.
//
// The reference's partial butterflies (ref: dct-generic.c:255-577) evaluate, per pass, the exact integer matrix
// product  dst[k*N + j] = (sum_i M[k][i] * src[j*N + i] + add) >> shift   (forward, result TRUNCATED to int16) and
//          dst[j*N + k] = clip16((sum_i M[i][k] * src[i*N + j] + add) >> shift)   (inverse).
// Integer addition is associative, so a plain dot product reproduces them bit for bit.
#pragma once
#include "common.cuh"
#include "coeff_rules.h"

namespace kvzc {

using namespace kvzcoeff;

// C[m], m = 0..32: the HEVC core-transform coefficient list; M32[k][i] = sgn * C[fold((k*(2i+1)) mod 128)]
// (cosine symmetries C[64-m] = -C[m], C[128-m] = C[m]); the N-point matrix takes rows 0, 32/N, 2*32/N, ...
static __constant__ int8_t c_tr32[33] = { 64, 90, 90, 90, 89, 88, 87, 85, 83, 82, 80, 78, 75, 73, 70, 67, 64,
                                   61, 57, 54, 50, 46, 43, 38, 36, 31, 25, 22, 18, 13, 9, 4, 0 };
static __constant__ int8_t c_dst4[16] = { 29, 55, 74, 84, 74, 74, 0, -74, 84, -29, -74, 55, 55, -84, 74, -29 };

__device__ __forceinline__ int tr_coef(int n, bool dst, int k, int i)
{
  if (dst) return c_dst4[k * 4 + i];
  int m = ((k * (32 / n)) * (2 * i + 1)) & 127;
  if (m > 64) m = 128 - m;
  return m <= 32 ? (int)c_tr32[m] : -(int)c_tr32[64 - m];
}

// Fill `mat` (N*N int8, shared) so that mat[i*N + k] = M[k][i] when `transposed` (forward use) or M[i][k] (inverse).
__device__ __forceinline__ void load_matrix(int8_t *mat, int n, bool dst, bool transposed)
{
  for (int e = threadIdx.x; e < n * n; e += blockDim.x) {
    const int i = e / n, k = e % n;
    mat[e] = (int8_t)(transposed ? tr_coef(n, dst, k, i) : tr_coef(n, dst, i, k));
  }
}

// forward pass over `g` blocks stored back to back: dst[k*N+j] = (short)((sum_i M[k][i]*src[j*N+i] + add) >> shift)
// matT[i*N + k] = M[k][i]
__device__ __forceinline__ void fwd_pass(const int16_t *src, int16_t *dst, const int8_t *matT, int n, int g, int shift)
{
  const int add = 1 << (shift - 1);
  const int nn = n * n;
  for (int e = threadIdx.x; e < g * nn; e += blockDim.x) {
    const int blk = e / nn, r = e - blk * nn, j = r / n, k = r - j * n;
    const int16_t *s = src + blk * nn + j * n;
    int acc = 0;
#pragma unroll 4
    for (int i = 0; i < n; ++i) acc += (int)matT[i * n + k] * (int)s[i];
    dst[blk * nn + k * n + j] = (int16_t)((acc + add) >> shift);
  }
}

// inverse pass: dst[j*N+k] = clip16((sum_i M[i][k]*src[i*N+j] + add) >> shift);  mat[i*N + k] = M[i][k]
__device__ __forceinline__ void inv_pass(const int16_t *src, int16_t *dst, const int8_t *mat, int n, int g, int shift)
{
  const int add = 1 << (shift - 1);
  const int nn = n * n;
  for (int e = threadIdx.x; e < g * nn; e += blockDim.x) {
    const int blk = e / nn, r = e - blk * nn, j = r / n, k = r - j * n;
    const int16_t *s = src + blk * nn + j;
    int acc = 0;
#pragma unroll 4
    for (int i = 0; i < n; ++i) acc += (int)mat[i * n + k] * (int)s[i * n];
    dst[blk * nn + j * n + k] = (int16_t)clip3(-32768, 32767, (acc + add) >> shift);
  }
}

// ---- DP2A formulation used by the fused frame-pass kernels -------------------------------------------------------
// v[k][j] = sum_i A[k][i] * src[j*W + i] over a tile of 1024 coefficients (1024 / W^2 blocks back to back), with
// A = M (forward) or A = M^T (inverse, fed with the transposed input).  The |coefficients| <= 90 fit int8 and the
// data is int16, so one IDP2A does two exact multiply-adds; A is stored as 4-packed rows
// P[(i / 4) * W + k] = { A[k][i], A[k][i+1], A[k][i+2], A[k][i+3] } so lanes with consecutive k read consecutive
// words.  Each of the 256 threads owns a 2 (k) x 2 (j) output tile: 4 LDS + 8 IDP2A per 16 multiply-adds.
template <int W>
__device__ __forceinline__ void load_matrix_packed(uint32_t *P, bool dst, bool transposed)
{
  for (int e = threadIdx.x; e < W * W / 4; e += blockDim.x) {
    const int i4 = e / W, k = e % W;
    uint32_t v = 0;
#pragma unroll
    for (int b = 0; b < 4; ++b) {
      const int i = 4 * i4 + b;
      const int c = transposed ? tr_coef(W, dst, i, k) : tr_coef(W, dst, k, i);
      v |= (uint32_t)(c & 0xff) << (8 * b);
    }
    P[e] = v;
  }
}

// STORE_KJ: result stored at out[k*W + j] (what the next pass reads as "row k"), else at out[j*W + k].
// CLIP: clip to int16 (inverse passes) instead of truncating (forward passes).  blockDim.x == 256, tile = 1024.
template <int W, bool STORE_KJ, bool CLIP, int G = 1024 / (W * W)>
__device__ __forceinline__ void mat_pass_dp2a(const int16_t *src, int16_t *out, const uint32_t *P, int shift)
{
  constexpr int WW = W * W, ITEMS = WW / 4;              // 2x2 output tiles per block
  const int t = threadIdx.x;
  const int gb = t / ITEMS, r = t - gb * ITEMS;
  if (gb >= G) return;                                   // tiles smaller than 1024 samples leave threads idle
  const int kp = r % (W / 2), jp = r / (W / 2);
  const int k0 = 2 * kp, j0 = 2 * jp;
  const int16_t *s0 = src + gb * WW + j0 * W, *s1 = s0 + W;
  int a00 = 0, a01 = 0, a10 = 0, a11 = 0;                // a[k][j]
#pragma unroll
  for (int i4 = 0; i4 < W / 4; ++i4) {
    const uint2 m = *reinterpret_cast<const uint2 *>(P + i4 * W + k0);      // rows k0, k0+1, columns 4*i4 .. +3
    const uint2 x0 = *reinterpret_cast<const uint2 *>(s0 + 4 * i4);          // src[j0][4*i4 .. +3]
    const uint2 x1 = *reinterpret_cast<const uint2 *>(s1 + 4 * i4);
    a00 = __dp2a_lo((int)x0.x, (int)m.x, a00); a00 = __dp2a_hi((int)x0.y, (int)m.x, a00);
    a01 = __dp2a_lo((int)x1.x, (int)m.x, a01); a01 = __dp2a_hi((int)x1.y, (int)m.x, a01);
    a10 = __dp2a_lo((int)x0.x, (int)m.y, a10); a10 = __dp2a_hi((int)x0.y, (int)m.y, a10);
    a11 = __dp2a_lo((int)x1.x, (int)m.y, a11); a11 = __dp2a_hi((int)x1.y, (int)m.y, a11);
  }
  const int add = 1 << (shift - 1);
  auto fin = [&](int v) -> int { v = (v + add) >> shift; return CLIP ? clip3(-32768, 32767, v) : (int)(int16_t)v; };
  int16_t *o = out + gb * WW;
  if (STORE_KJ) {
    *reinterpret_cast<uint32_t *>(o + k0 * W + j0) = (uint32_t)(uint16_t)fin(a00) | ((uint32_t)(uint16_t)fin(a01) << 16);
    *reinterpret_cast<uint32_t *>(o + (k0 + 1) * W + j0) = (uint32_t)(uint16_t)fin(a10) | ((uint32_t)(uint16_t)fin(a11) << 16);
  } else {
    *reinterpret_cast<uint32_t *>(o + j0 * W + k0) = (uint32_t)(uint16_t)fin(a00) | ((uint32_t)(uint16_t)fin(a10) << 16);
    *reinterpret_cast<uint32_t *>(o + (j0 + 1) * W + k0) = (uint32_t)(uint16_t)fin(a01) | ((uint32_t)(uint16_t)fin(a11) << 16);
  }
}

__device__ __forceinline__ int ilog2(int n) { return 31 - __clz(n); }

// ---- quantisation ---------------------------------------------------------------------------
static __constant__ int c_quant_scales[6] = { COEFF_QUANT_SCALES };
static __constant__ int c_inv_quant_scales[6] = { COEFF_INV_QUANT_SCALES };

// position of scan index `idx` for an n x n block (ref: tables.c kvz_g_sig_last_scan): 4x4 coefficient groups
// visited in scan order (scan_small), same order inside a group
__device__ __forceinline__ int scan_pos(int scan_idx, int log2_n, int idx)
{
  if (log2_n <= 2) return scan_small(scan_idx, log2_n, idx);
  const int n = 1 << log2_n;
  const int cg = scan_small(scan_idx, log2_n - 2, idx >> 4);                  // group (y*(n/4) + x)
  const int in = scan_small(scan_idx, 2, idx & 15);
  const int gw = n >> 2;
  return ((cg / gw) * 4 + (in >> 2)) * n + (cg % gw) * 4 + (in & 3);
}

// raster positions of the 16 scan positions of coefficient group g (quant_sign_hiding's scan), in registers
__device__ __forceinline__ void group_scan(int pos[16], int scan_idx, int log2_n, int g)
{
#pragma unroll
  for (int k = 0; k < 16; ++k) pos[k] = scan_pos(scan_idx, log2_n, g * 16 + k);
}

struct QuantConsts {
  int qc, q_bits, add, q_bits8;
};
__device__ __forceinline__ QuantConsts quant_consts(const kvz_cuda_quant_params &p, int log2_n, int type)
{
  QuantConsts c;
  const int qp_scaled = scaled_qp(type, p.qp, (p.bitdepth - 8) * 6);
  c.qc = c_quant_scales[qp_scaled % 6];
  const int transform_shift = 15 - p.bitdepth - log2_n;
  c.q_bits = 14 + qp_scaled / 6 + transform_shift;
  c.add = (p.slice_is_intra ? 171 : 85) << (c.q_bits - 9);
  c.q_bits8 = c.q_bits - 8;
  return c;
}

// kvz_quant (ref: quant-generic.c:50-180) for ONE n x n block held in shared memory.
// coef -> q (both shared, n*n); delta_u: n*n int32 shared scratch; all threads of the CTA participate.
__device__ __forceinline__ void quant_block(const kvz_cuda_quant_params &p, const int16_t *coef, int16_t *q,
                                            int32_t *delta_u, int n, int type, int scan_idx)
{
  const int log2_n = ilog2(n);
  const QuantConsts c = quant_consts(p, log2_n, type);
  int ac = 0;
  for (int e = threadIdx.x; e < n * n; e += blockDim.x) {
    const int level_in = coef[e];
    const long long abs_level = abs(level_in);
    int level = (int)((abs_level * c.qc + c.add) >> c.q_bits);
    ac += level;
    delta_u[e] = (int)((abs_level * c.qc - ((long long)level << c.q_bits)) >> c.q_bits8);
    level = level_in < 0 ? -level : level;
    q[e] = (int16_t)clip3(-32768, 32767, level);
  }
  ac = block_sum(ac);
  __shared__ int s_ac;
  __shared__ int s_cg_nz[64];
  if (threadIdx.x == 0) s_ac = ac;
  const int num_cg = (n * n) >> 4;
  // per coefficient-group "has a non-zero" flags (before any sign hiding), in scan order
  for (int g = threadIdx.x; g < num_cg; g += blockDim.x) {
    int nz = 0;
    for (int k = 0; k < 16; ++k) nz |= q[scan_pos(scan_idx, log2_n, g * 16 + k)] != 0;
    s_cg_nz[g] = nz;
  }
  __syncthreads();
  if (!p.signhide_enable || s_ac < 2) return;
  // one thread per coefficient group: the groups only interact through "is this the last non-zero group"
  for (int g = threadIdx.x; g < num_cg; g += blockDim.x) {
    if (!s_cg_nz[g]) continue;
    int pos[16];
    group_scan(pos, scan_idx, log2_n, g);
    quant_sign_hiding(pos, coef, q, delta_u, s_cg_nz, num_cg, g);
  }
  __syncthreads();
}

// kvz_dequant (ref: quant-generic.c:298-340), flat scaling lists, one n x n block in shared memory
__device__ __forceinline__ void dequant_block(const kvz_cuda_quant_params &p, const int16_t *q, int16_t *coef, int n,
                                              int type)
{
  const int transform_shift = 15 - p.bitdepth - ilog2(n);
  const int qp_scaled = scaled_qp(type, p.qp, (p.bitdepth - 8) * 6);
  const int shift = 20 - 14 - transform_shift;
  const int scale = c_inv_quant_scales[qp_scaled % 6] << (qp_scaled / 6);
  const int add = 1 << (shift - 1);
  for (int e = threadIdx.x; e < n * n; e += blockDim.x)
    coef[e] = (int16_t)clip3(-32768, 32767, ((int)q[e] * scale + add) >> shift);
}

// runtime-width dispatch onto the templated DP2A passes (one TU, 256-thread CTA)
__device__ __forceinline__ void load_packed_any(uint32_t *P, int n, bool dst, bool transposed)
{
  if (n == 4) load_matrix_packed<4>(P, dst, transposed);
  else if (n == 8) load_matrix_packed<8>(P, dst, transposed);
  else if (n == 16) load_matrix_packed<16>(P, dst, transposed);
  else load_matrix_packed<32>(P, dst, transposed);
}
template <bool STORE_KJ, bool CLIP>
__device__ __forceinline__ void pass_any(const int16_t *src, int16_t *out, const uint32_t *P, int n, int shift)
{
  if (n == 4) mat_pass_dp2a<4, STORE_KJ, CLIP, 1>(src, out, P, shift);
  else if (n == 8) mat_pass_dp2a<8, STORE_KJ, CLIP, 1>(src, out, P, shift);
  else if (n == 16) mat_pass_dp2a<16, STORE_KJ, CLIP, 1>(src, out, P, shift);
  else mat_pass_dp2a<32, STORE_KJ, CLIP, 1>(src, out, P, shift);
}

// ---- kvz_quantize_residual for one TU, all threads of the CTA (ref: quant-generic.c:198-292, RDOQ-off branch) ----
struct TuScratch {
  __align__(16) int16_t a[32 * 32];
  __align__(16) int16_t b[32 * 32];
  __align__(16) int16_t q[32 * 32];
  int32_t d[32 * 32];
  __align__(16) int8_t m[32 * 32];      // 4-packed transform matrix (32 * 32 / 4 words)
  int has;
};

// ref/pred/rec point at the TU's top-left sample; pred may live in shared memory (pred_stride = width).
// phase: 0 whole function, 1 residual + forward transform only, 2 dequant + inverse + reconstruction only.
// Returns has_coeffs (0 for phase 1).
template <class T>
__device__ __forceinline__ int quantize_residual_tu(TuScratch &s, const kvz_cuda_quant_params &p, int n, int color,
                                                    int scan_idx, bool use_trskip, bool cu_is_intra, bool early_skip,
                                                    int phase, const T *ref, int ref_stride, const T *pred,
                                                    int pred_stride, T *rec, int rec_stride, int16_t *coeff_out)
{
  constexpr int PIXMAX = (1 << PixTraits<T>::bd) - 1;
  const int nn = n * n, l2 = ilog2(n);
  const bool use_dst = (n == 4 && color == 0 && cu_is_intra);      // ref: strategies-dct.c:78-96
  const int ts_shift = 15 - p.bitdepth - l2;                        // ref: transform.c:150-185
  if (threadIdx.x == 0) s.has = 0;
  if (phase != 2) {
    for (int e = threadIdx.x; e < nn; e += blockDim.x) {
      const int y = e / n, x = e - y * n;
      s.a[e] = (int16_t)((int)ref[y * ref_stride + x] - (int)pred[y * pred_stride + x]);
    }
    if (!use_trskip) load_packed_any(reinterpret_cast<uint32_t *>(s.m), n, use_dst, false);
    __syncthreads();
    if (use_trskip) {
      for (int e = threadIdx.x; e < nn; e += blockDim.x) s.b[e] = (int16_t)((uint16_t)s.a[e] << ts_shift);
    } else {
      pass_any<true, false>(s.a, s.q, reinterpret_cast<const uint32_t *>(s.m), n, l2 - 1 + (p.bitdepth - 8));
      __syncthreads();
      pass_any<true, false>(s.q, s.b, reinterpret_cast<const uint32_t *>(s.m), n, l2 + 6);
    }
    __syncthreads();
    if (phase == 1) {   // the host runs kvz_rdoq on these coefficients
      for (int e = threadIdx.x; e < nn; e += blockDim.x) coeff_out[e] = s.b[e];
      return 0;
    }
    quant_block(p, s.b, s.q, s.d, n, color == 0 ? 0 : 2, scan_idx);
    __syncthreads();
  } else {
    for (int e = threadIdx.x; e < nn; e += blockDim.x) s.q[e] = coeff_out[e];
    __syncthreads();
  }
  int any = 0;
  for (int e = threadIdx.x; e < nn; e += blockDim.x) {
    const int16_t v = s.q[e];
    if (phase == 0) coeff_out[e] = v;
    any |= v != 0;
  }
  if (any) atomicOr(&s.has, 1);
  __syncthreads();
  const int has = s.has;
  if (has && !early_skip) {
    dequant_block(p, s.q, s.b, n, color == 0 ? 0 : (color == 1 ? 2 : 3));
    __syncthreads();
    if (use_trskip) {
      const int off = 1 << (ts_shift - 1);
      for (int e = threadIdx.x; e < nn; e += blockDim.x) s.a[e] = (int16_t)(((int)s.b[e] + off) >> ts_shift);
    } else {
      // inverse = the same DP2A passes with A = M^T on the transposed coefficients (see mat_pass_dp2a)
      for (int e = threadIdx.x; e < nn; e += blockDim.x) { const int y = e / n, x = e - y * n; s.q[x * n + y] = s.b[e]; }
      load_packed_any(reinterpret_cast<uint32_t *>(s.m), n, use_dst, true);
      __syncthreads();
      pass_any<true, true>(s.q, s.b, reinterpret_cast<const uint32_t *>(s.m), n, 7);
      __syncthreads();
      pass_any<false, true>(s.b, s.a, reinterpret_cast<const uint32_t *>(s.m), n, 12 - (p.bitdepth - 8));
    }
    __syncthreads();
    for (int e = threadIdx.x; e < nn; e += blockDim.x) {
      const int y = e / n, x = e - y * n;
      const int16_t val = (int16_t)(s.a[e] + (int)pred[y * pred_stride + x]);
      rec[y * rec_stride + x] = (T)clip3(0, PIXMAX, (int)val);
    }
  } else if ((const void *)rec != (const void *)pred) {
    for (int e = threadIdx.x; e < nn; e += blockDim.x) {
      const int y = e / n, x = e - y * n;
      rec[y * rec_stride + x] = pred[y * pred_stride + x];
    }
  }
  return has;
}

}  // namespace kvzc
