// framepass.cu -- the frame-level hot-path pass: every strategy kernel an all-intra encode of one frame calls,
// batched over all CTUs of the frame and evaluated for every quadtree depth, with the frame resident in HBM.
//
// Per I420 frame (W x H luma, 8-bit), for depth d = 0..3 (luma block width w = 32,16,8,4):
//   1. rough search      : 35 intra modes x every w x w block -> SATD costs      (search_intra_rough, search_intra.c:391-530)
//   2. mode selection    : first minimum of the 35 costs
//   3. luma recon        : refs -> prediction of the chosen mode -> residual -> DCT/DST -> quant -> dequant -> IDCT
//                          -> reconstruction, coefficients, has_coeffs, SSD        (kvz_intra_recon_cu, intra.c:623-698 with
//                          kvz_quantize_residual's RDOQ-off branch, quant-generic.c:198-292; kvz_pixels_calc_ssd)
//   4. chroma recon      : same for U and V with w/2 blocks and the co-located luma mode (d = 0..2)
// then on the 8x8-level reconstruction:
//   4b. deblocking       : every 8x8 edge of that uniform intra quadtree, luma + chroma, in place
//                          (kvz_filter_deblock_lcu, filter.c:783-792; csrc/deblock.cu)
//   5. SAO               : edge statistics (4 classes), offsets, edge / band delta-distortion, reconstruction per CTU
//                          (sao_search_*, sao.c:605-669 and kvz_sao_reconstruct, sao.c:302-361 call shapes)
//   6. picture checksum  : array_checksum of the three SAO-filtered planes          (nal.c:77-86)
// Prediction references come from a caller-supplied reconstruction (rec_in); passing the source itself gives the
// open-loop variant used for benchmarking.  The closed-loop CTU-serial search driver is the next scope row
// (SURVEY.md 8f rank 2) -- this pass is the data-parallel part underneath it.
#include <vector>

#include "common.cuh"
#include "intra.cuh"
#include "transform.cuh"

namespace kvzc {

int rough_search_u8(int log2w, const uint8_t *src, const uint8_t *rec, int stride, int pic_w, int pic_h, uint32_t *costs,
                    int8_t *best_mode, uint32_t *best_cost, cudaStream_t st);
int rough_search_u16(int log2w, const uint16_t *src, const uint16_t *rec, int stride, int pic_w, int pic_h, uint32_t *costs,
                     int8_t *best_mode, uint32_t *best_cost, cudaStream_t st);

// kvz_intra_recon_cu for a tile of 1024 samples (G = 1024 / W^2 TUs of one colour plane) per 256-thread CTA:
// references -> prediction of the chosen mode -> residual -> DCT/DST -> quant (+ sign hiding) -> dequant -> inverse
// -> reconstruction, SSD.  All TUs walk the same barrier sequence; data-dependent decisions (has_coeffs,
// ac_sum < 2) are predicates.  Transforms use the DP2A matrix passes of transform.cuh.
// INTER = true: the same walk for an inter CU's TU grid -- rec_in is then the motion-compensated PREDICTION plane,
// modes is unused, the scan is diagonal, no DST, and has_out is an int32 array (inter pass blob layout).
// PHASE splits the walk around kvz_rdoq (quant-generic.c:234-240): 0 = whole function with kvz_quant; 1 = up to the
// forward transform (coefficients -> coeff); 2 = from the quantised levels in coeff (written by rdoq_grid) onwards.
// TRSKIP (4x4 luma only): transform skip instead of the DST (kvz_transformskip / kvz_itransformskip, transform.c:150-185).
template <class T, int LOG2W, bool INTER = false, int PHASE = 0, bool TRSKIP = false>
__global__ void __launch_bounds__(256) intra_recon_kernel(kvz_cuda_quant_params p, const T *__restrict__ src,
                                                          const T *__restrict__ rec_in, int stride, int pic_w, int pic_h,
                                                          int color, int blocks_x, int nblk,
                                                          const int8_t *__restrict__ modes, T *__restrict__ rec_out,
                                                          int16_t *__restrict__ coeff, uint8_t *__restrict__ has_out,
                                                          uint32_t *__restrict__ ssd_out)
{
  constexpr int W = 1 << LOG2W, WW = W * W, NREF = 2 * W + 1;
  constexpr int E = 1024, G = E / WW;               // 1, 4, 16, 64 TUs per CTA
  constexpr int PIXMAX = (1 << PixTraits<T>::bd) - 1;
  constexpr int NCG = WW / 16;                      // coefficient groups per TU
  __shared__ __align__(16) int16_t s_a[E], s_b[E], s_q[E];
  __shared__ int32_t s_d[E];
  __shared__ __align__(16) uint32_t s_pf[WW / 4], s_pi[WW / 4];
  __shared__ T s_ref[G][4][NREF + 3];
  __shared__ T s_pred[E];
  __shared__ int s_dc[G], s_has[G], s_ac[G], s_ssd[G];
  __shared__ int8_t s_mode[G];
  __shared__ uint8_t s_cgnz[G][NCG];
  __shared__ BuildRefCtx s_ctx[G];
  const int is_c = color != 0;
  const int first = blockIdx.x * G;
  const int l2 = LOG2W;
  const bool use_dst = (!INTER && W == 4 && color == 0);                // intra luma 4x4, ref: strategies-dct.c:78-96

  // ---- references, smoothed references, DC, mode
  for (int gb = threadIdx.x; gb < G; gb += blockDim.x) {
    const int b = min(first + gb, nblk - 1);
    if (!INTER && PHASE != 2) s_ctx[gb] = build_ref_ctx(LOG2W, color, ((b % blocks_x) * W) << is_c, ((b / blocks_x) * W) << is_c, pic_w, pic_h);
    s_mode[gb] = (!INTER && first + gb < nblk) ? modes[first + gb] : 0;
    s_has[gb] = 0; s_ac[gb] = 0; s_ssd[gb] = 0;
  }
  load_matrix_packed<W>(s_pf, use_dst, false);
  load_matrix_packed<W>(s_pi, use_dst, true);
  __syncthreads();
  if (!INTER && PHASE != 2) {
  for (int e = threadIdx.x; e < G * 2 * NREF; e += blockDim.x) {
    const int gb = e / (2 * NREF), r = e - gb * 2 * NREF;
    const bool is_top = r < NREF;
    const int k = is_top ? r : r - NREF;
    s_ref[gb][is_top ? 0 : 1][k] = (T)build_ref_entry(s_ctx[gb], rec_in, stride, is_top, k);
  }
  __syncthreads();
  for (int e = threadIdx.x; e < G * 2 * NREF; e += blockDim.x) {
    const int gb = e / (2 * NREF), r = e - gb * 2 * NREF;
    const bool is_top = r < NREF;
    const int k = is_top ? r : r - NREF;
    s_ref[gb][is_top ? 2 : 3][k] = (T)ref_smooth_entry(s_ref[gb][0], s_ref[gb][1], is_top, k, NREF);
  }
  for (int gb = threadIdx.x; gb < G; gb += blockDim.x) s_dc[gb] = dc_value(LOG2W, s_ref[gb][0], s_ref[gb][1]);
  __syncthreads();
  }

  // ---- prediction and residual
  for (int e = threadIdx.x; e < E; e += blockDim.x) {
    const int gb = e / WW, r = e - gb * WW, y = r >> LOG2W, x = r & (W - 1), b = first + gb;
    int pv = 0, sv = 0;
    if (b < nblk) {
      const long off = (long)((b / blocks_x) * W + y) * stride + (b % blocks_x) * W + x;
      if (INTER) pv = rec_in[off];
      else if (PHASE == 2) pv = rec_out[off];          // the forward half parked the prediction in the reconstruction plane
      else pv = intra_predict_px<T>(RefView<T>{ s_ref[gb][0], s_ref[gb][1], s_ref[gb][2], s_ref[gb][3], s_dc[gb] }, LOG2W, s_mode[gb], color, true, x, y);
      sv = src[off];
      if (PHASE == 1) rec_out[off] = (T)pv;
    }
    s_pred[e] = (T)pv;
    s_a[e] = (int16_t)(sv - pv);
    if (PHASE == 2) s_q[e] = b < nblk ? coeff[(size_t)b * WW + r] : (int16_t)0;
  }
  __syncthreads();

  if (PHASE != 2) {
  // ---- forward transform (ref: dct-generic.c:579-588, 611-619): tmp[k][j], then coef[k][j]
  if constexpr (TRSKIP) {
    const int ts_shift = 15 - p.bitdepth - l2;
    for (int e = threadIdx.x; e < E; e += blockDim.x) s_b[e] = (int16_t)((uint16_t)s_a[e] << ts_shift);
  } else {
    mat_pass_dp2a<W, true, false>(s_a, s_q, s_pf, l2 - 1 + (p.bitdepth - 8));
    __syncthreads();
    mat_pass_dp2a<W, true, false>(s_q, s_b, s_pf, l2 + 6);
  }
  __syncthreads();
  if (PHASE == 1) {
    for (int e = threadIdx.x; e < E; e += blockDim.x) {
      const int gb = e / WW, r = e - gb * WW, b = first + gb;
      if (b < nblk) coeff[(size_t)b * WW + r] = s_b[e];
    }
    return;
  }

  // ---- quantisation (ref: quant-generic.c:50-180)
  const QuantConsts qc = quant_consts(p, l2, is_c ? 2 : 0);
  for (int e = threadIdx.x; e < E; e += blockDim.x) {
    const int gb = e / WW;
    const int level_in = s_b[e];
    const long long abs_level = abs(level_in);
    int level = (int)((abs_level * qc.qc + qc.add) >> qc.q_bits);
    s_d[e] = (int)((abs_level * qc.qc - ((long long)level << qc.q_bits)) >> qc.q_bits8);
    if (p.signhide_enable && level) atomicAdd(&s_ac[gb], level);
    level = level_in < 0 ? -level : level;
    s_q[e] = (int16_t)clip3(-32768, 32767, level);
  }
  __syncthreads();
  if (p.signhide_enable) {
    for (int i = threadIdx.x; i < G * NCG; i += blockDim.x) {
      const int gb = i / NCG, cg = i - gb * NCG;
      const int mode = s_mode[gb];
      const int scan = ((!is_c && W <= 8) || (is_c && W == 4)) ? ((mode >= 6 && mode <= 14) ? 2 : ((mode >= 22 && mode <= 30) ? 1 : 0)) : 0;
      int nz = 0;
      for (int k = 0; k < 16; ++k) nz |= s_q[gb * WW + scan_pos(scan, l2, cg * 16 + k)] != 0;
      s_cgnz[gb][cg] = (uint8_t)nz;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < G * NCG; i += blockDim.x) {
      const int gb = i / NCG, cg = i - gb * NCG;
      if (s_ac[gb] < 2 || !s_cgnz[gb][cg]) continue;
      const int mode = s_mode[gb];
      const int scan = ((!is_c && W <= 8) || (is_c && W == 4)) ? ((mode >= 6 && mode <= 14) ? 2 : ((mode >= 22 && mode <= 30) ? 1 : 0)) : 0;
      int pos[16];
      group_scan(pos, scan, l2, cg);
      quant_sign_hiding(pos, s_b + gb * WW, s_q + gb * WW, s_d + gb * WW, s_cgnz[gb], NCG, cg);
    }
    __syncthreads();
  }
  }  // PHASE != 2

  // ---- coefficients out, has_coeffs, dequant (ref: quant-generic.c:298-340) into the TRANSPOSED layout the
  //      inverse passes consume
  {
    const int transform_shift = 15 - p.bitdepth - l2;
    const int qp_scaled = scaled_qp(is_c ? (color == 1 ? 2 : 3) : 0, p.qp, (p.bitdepth - 8) * 6);
    const int shift = 20 - 14 - transform_shift;
    const int scale = c_inv_quant_scales[qp_scaled % 6] << (qp_scaled / 6);
    const int add = 1 << (shift - 1);
    for (int e = threadIdx.x; e < E; e += blockDim.x) {
      const int gb = e / WW, r = e - gb * WW, y = r >> LOG2W, x = r & (W - 1), b = first + gb;
      const int16_t v = s_q[e];
      if (b < nblk) {
        if (PHASE != 2) coeff[(size_t)b * WW + r] = v;
        if (v != 0) s_has[gb] = 1;
      }
      const int dq = clip3(-32768, 32767, ((int)v * scale + add) >> shift);
      if constexpr (TRSKIP) { const int ts_shift = 15 - p.bitdepth - l2; s_b[e] = (int16_t)((dq + (1 << (ts_shift - 1))) >> ts_shift); }
      else s_b[gb * WW + x * W + y] = (int16_t)dq;
    }
  }
  __syncthreads();
  // ---- inverse transform (ref: dct-generic.c:590-599, 621-629)
  if constexpr (!TRSKIP) {
    mat_pass_dp2a<W, true, true>(s_b, s_a, s_pi, 7);
    __syncthreads();
    mat_pass_dp2a<W, false, true>(s_a, s_b, s_pi, 12 - (p.bitdepth - 8));
    __syncthreads();
  }

  // ---- reconstruction + SSD (ref: quant-generic.c:263-292, picture-generic.c:536-551)
  for (int e = threadIdx.x; e < E; e += blockDim.x) {
    const int gb = e / WW, r = e - gb * WW, y = r >> LOG2W, x = r & (W - 1), b = first + gb;
    int sq = 0;
    if (b < nblk) {                                   // (no early exit: every lane takes part in the shuffles below)
      const int pv = s_pred[e];
      int rv = pv;
      if (s_has[gb]) rv = clip3(0, PIXMAX, (int)(int16_t)(s_b[e] + pv));
      const long off = (long)((b / blocks_x) * W + y) * stride + (b % blocks_x) * W + x;
      rec_out[off] = (T)rv;
      const int dv = (int)src[off] - rv;
      sq = dv * dv;
    }
    // reduce within the lanes of this warp that belong to the same TU, then one atomic per TU per warp
    constexpr int SEG = WW < 32 ? WW : 32;
#pragma unroll
    for (int o = SEG / 2; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
    if ((threadIdx.x & (SEG - 1)) == 0) atomicAdd(&s_ssd[gb], sq);
  }
  __syncthreads();
  for (int gb = threadIdx.x; gb < G; gb += blockDim.x)
    if (first + gb < nblk) {
      if (INTER) reinterpret_cast<int32_t *>(has_out)[first + gb] = s_has[gb];
      else has_out[first + gb] = (uint8_t)s_has[gb];
      ssd_out[first + gb] = (uint32_t)(s_ssd[gb] >> (2 * (PixTraits<T>::bd - 8)));
    }
}

template <class T>
struct SaoPlanesT {
  const T *src[3];
  const T *rec[3];
  T *out[3];
  int Wp[3], Hp[3];
};
using SaoPlanes = SaoPlanesT<uint8_t>;

// One CTA per (plane, CTU): ONE pass over the CTU gathers the edge statistics of all four classes
// (calc_sao_edge_dir, ref: sao-generic.c:50-81) and the per-band sums; everything else follows in closed form:
//   offsets[k]      = clip(sum_k / cnt_k)                                   (the pass's decision rule)
//   edge ddist      = sum_k (o_k^2 * cnt_k - 2 * o_k * sum_k)               == sum_i ((d_i - o)^2 - d_i^2), the value
//                     kvz_sao_edge_ddistortion accumulates pixel by pixel (ref: sao_shared_generics.h:52-91)
//   band ddist      = the same identity over the four bands                 (ref: sao_shared_generics.h:93-130)
// so the delta-distortion "kernels" cost nothing on the device.  Above 8 bits the edge statistics and the edge
// delta-distortion both work on the rounded difference (d + 2^(bd-9)) >> (bd-8) (sao-generic.c:66,77,
// sao_shared_generics.h:64,83); the band distortion uses the raw difference.
template <class T>
__global__ void __launch_bounds__(256) sao_ctu_kernel(SaoPlanesT<T> pl, int nctu, int ctus_x, int32_t *__restrict__ stats,
                                                      int32_t *__restrict__ dd, int32_t *__restrict__ band_dd,
                                                      int8_t *__restrict__ best, int32_t *__restrict__ dec_off,
                                                      uint32_t *__restrict__ cksum_scratch)
{
  constexpr int BD = PixTraits<T>::bd;
  __shared__ int s_acc[4][2][5];
  __shared__ int s_band[2][4];
  const int i = blockIdx.x, color = i / nctu, ctu = i - color * nctu;
  const int Wp = pl.Wp[color], Hp = pl.Hp[color], lw = color ? 32 : 64;
  const int x0 = (ctu % ctus_x) * lw, y0 = (ctu / ctus_x) * lw;
  const int bw = min(lw, Wp - x0), bh = min(lw, Hp - y0);
  const T *orig = pl.src[color] + (long)y0 * Wp + x0, *rec = pl.rec[color] + (long)y0 * Wp + x0;
  const int bp = (i * 7) % 29;
  if (i == 0 && threadIdx.x < 6) cksum_scratch[threadIdx.x] = 0;
  for (int t = threadIdx.x; t < 48; t += blockDim.x) { if (t < 40) (&s_acc[0][0][0])[t] = 0; else (&s_band[0][0])[t - 40] = 0; }
  __syncthreads();
  // Per-thread accumulators are packed (a thread sees at most 16 samples of the CTU): counts in 6-bit fields, sums of
  // the (rounded) differences as arithmetic 16-bit lane pairs (|sum| <= 16 * 256) -- 19 registers instead of 48, which
  // doubles the number of resident CTAs.
  uint32_t cntp[4] = { 0, 0, 0, 0 }, bcp = 0;
  int sump[4][3], bsp[2] = { 0, 0 };
#pragma unroll
  for (int e = 0; e < 4; ++e) { sump[e][0] = 0; sump[e][1] = 0; sump[e][2] = 0; }
  for (int t = threadIdx.x; t < bw * bh; t += blockDim.x) {
    const int y = t / bw, x = t - y * bw;
    const int c = rec[(long)y * Wp + x];
    const int diff = (int)orig[(long)y * Wp + x] - c;
    const int diffr = BD > 8 ? (diff + (1 << (BD > 8 ? BD - 9 : 0))) >> (BD - 8) : diff;
    const int band = (c >> (BD - 5)) - bp;
    if (band >= 0 && band < 4) {
      bcp += 1u << (6 * band);
      const int v = diff * ((band & 1) ? 65536 : 1);
      bsp[0] += band < 2 ? v : 0;
      bsp[1] += band >= 2 ? v : 0;
    }
    if (x >= 1 && y >= 1 && x < bw - 1 && y < bh - 1) {        // the strategies only see the block: no outside neighbours
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        int ax, ay;
        sao_eo_offsets(e, ax, ay);
        const int cat = sao_eo_cat(rec[(long)(y + ay) * Wp + x + ax], rec[(long)(y - ay) * Wp + x - ax], c);
        cntp[e] += 1u << (6 * cat);
        const int v = diffr * ((cat & 1) ? 65536 : 1);
        sump[e][0] += cat < 2 ? v : 0;
        sump[e][1] += (cat >> 1) == 1 ? v : 0;
        sump[e][2] += cat == 4 ? diffr : 0;
      }
    }
  }
  auto lane_lo = [](int x) { return (int)(short)x; };
  auto lane_hi = [](int x) { return (x - (int)(short)x) >> 16; };
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const int bsum = (e & 1) ? lane_hi(bsp[e >> 1]) : lane_lo(bsp[e >> 1]);
    const int b1 = warp_sum(bsum), b2 = warp_sum((int)((bcp >> (6 * e)) & 63));
    if ((threadIdx.x & 31) == 0) { atomicAdd(&s_band[0][e], b1); atomicAdd(&s_band[1][e], b2); }
#pragma unroll
    for (int k = 0; k < 5; ++k) {
      const int sk = k == 4 ? sump[e][2] : ((k & 1) ? lane_hi(sump[e][k >> 1]) : lane_lo(sump[e][k >> 1]));
      const int v1 = warp_sum(sk), v2 = warp_sum((int)((cntp[e] >> (6 * k)) & 63));
      if ((threadIdx.x & 31) == 0) { atomicAdd(&s_acc[e][0][k], v1); atomicAdd(&s_acc[e][1][k], v2); }
    }
  }
  __syncthreads();
  for (int t = threadIdx.x; t < 40; t += blockDim.x) stats[(size_t)i * 40 + t] = (&s_acc[0][0][0])[t];
  if (threadIdx.x == 0) {
    const int n3 = 3 * nctu;
    int be = 0, bd = 0, off_best[5] = { 0, 0, 0, 0, 0 };
    for (int e = 0; e < 4; ++e) {
      int o[5], v = 0;
      o[0] = 0;
      for (int k = 1; k < 5; ++k) o[k] = s_acc[e][1][k] ? clip3(-7, 7, s_acc[e][0][k] / s_acc[e][1][k]) : 0;
      for (int k = 1; k < 5; ++k) v += o[k] * o[k] * s_acc[e][1][k] - 2 * o[k] * s_acc[e][0][k];
      dd[(size_t)e * n3 + i] = v;
      if (e == 0 || v < bd) { bd = v; be = e; for (int k = 0; k < 5; ++k) off_best[k] = o[k]; }
    }
    const int bands[4] = { 1, -1, 2, -2 };
    int bv = 0;
    for (int k = 0; k < 4; ++k) bv += bands[k] * bands[k] * s_band[1][k] - 2 * bands[k] * s_band[0][k];
    band_dd[i] = bv;
    best[i] = (int8_t)(bd < 0 ? be : -1);
    for (int k = 0; k < 5; ++k) dec_off[(size_t)i * 5 + k] = off_best[k];
  }
}

// sao_reconstruct_color (edge type) of the chosen class for every CTU of the three planes; pixels on the picture
// border (no neighbours) and CTUs without SAO are copied (ref: sao-generic.c:84-124, sao.c:302-361 call shape).
template <class T>
__global__ void __launch_bounds__(256) sao_apply_kernel(SaoPlanesT<T> pl, int nctu, int ctus_x, const int8_t *__restrict__ best,
                                                        const int32_t *__restrict__ dec_off)
{
  const int i = blockIdx.x, color = i / nctu, ctu = i - color * nctu;
  const int Wp = pl.Wp[color], Hp = pl.Hp[color], lw = color ? 32 : 64;
  const int x0 = (ctu % ctus_x) * lw, y0 = (ctu / ctus_x) * lw;
  const int bw = min(lw, Wp - x0), bh = min(lw, Hp - y0);
  const T *rec = pl.rec[color];
  T *out = pl.out[color];
  const int eo = best[i];
  EdgeOffsets off;
#pragma unroll
  for (int k = 0; k < 5; ++k) off.o[k] = dec_off[(size_t)i * 5 + k];
  int ax = 0, ay = 0;
  if (eo >= 0) sao_eo_offsets(eo, ax, ay);
  for (int t = threadIdx.x; t < bw * bh; t += blockDim.x) {
    const int y = y0 + t / bw, x = x0 + t % bw;
    const long o = (long)y * Wp + x;
    int v = rec[o];
    if (eo >= 0 && x >= 1 && y >= 1 && x < Wp - 1 && y < Hp - 1)
      v = sao_edge_px(v, rec[o + (long)ay * Wp + ax], rec[o - (long)ay * Wp - ax], PixTraits<T>::bd, off);
    out[o] = (T)v;
  }
}

// picture checksum of the three planes in one launch (ref: nal-generic.c:57-82); blockIdx.y = plane
__global__ void __launch_bounds__(256) checksum3_kernel(SaoPlanes pl, uint32_t *__restrict__ scratch, uint8_t *__restrict__ out12)
{
  const int color = blockIdx.y;
  const int Wp = pl.Wp[color], Hp = pl.Hp[color];
  const uint8_t *data = pl.out[color];
  uint32_t s = 0;
  const int total4 = Wp * Hp / 4;                      // widths are multiples of 4: four pixels of one row per word
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < total4; t += gridDim.x * blockDim.x) {
    const int p = t * 4, y = p / Wp, x = p - y * Wp;
    const uint32_t v = *reinterpret_cast<const uint32_t *>(data + p);
    const uint32_t m0 = (uint32_t)((x & 0xff) ^ (y & 0xff) ^ (x >> 8) ^ (y >> 8)) & 0xff;   // x, x+1, x+2, x+3 share x >> 8
    const uint32_t mask = m0 | ((m0 ^ 1u) << 8) | ((m0 ^ 2u) << 16) | ((m0 ^ 3u) << 24);  // x & 3 == 0
    s = __dp4a(v ^ mask, 0x01010101u, s);
  }
  s = (uint32_t)block_sum((int)s);
  __shared__ bool s_last;
  if (threadIdx.x == 0) {
    atomicAdd(&scratch[2 * color], s);
    __threadfence();
    s_last = atomicAdd(&scratch[2 * color + 1], 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (s_last && threadIdx.x == 0) {
    const uint32_t t = atomicAdd(&scratch[2 * color], 0u);
    out12[4 * color + 0] = (uint8_t)(t >> 24); out12[4 * color + 1] = (uint8_t)(t >> 16);
    out12[4 * color + 2] = (uint8_t)(t >> 8); out12[4 * color + 3] = (uint8_t)t;
  }
}

// ---- compact form of the coefficient region: bitmap of non-zero 32-byte chunks + the chunks themselves, in order.
// Three small launches: per-tile (1024 chunks) counts, exclusive scan of the tile counts, ordered write.
constexpr int CMP_TILE = 1024;
__device__ __forceinline__ bool chunk_nonzero(const uint4 *p) { const uint4 a = p[0], b = p[1]; return (a.x | a.y | a.z | a.w | b.x | b.y | b.z | b.w) != 0; }

__global__ void __launch_bounds__(256) compact_count_kernel(const uint4 *__restrict__ region, uint32_t n_chunks, uint32_t *__restrict__ tile_counts)
{
  __shared__ int s_cnt;
  if (threadIdx.x == 0) s_cnt = 0;
  __syncthreads();
  int mine = 0;
  for (int k = 0; k < CMP_TILE / 256; ++k) {
    const uint32_t c = blockIdx.x * CMP_TILE + k * 256 + threadIdx.x;
    if (c < n_chunks && chunk_nonzero(region + 2 * (size_t)c)) ++mine;
  }
  mine = warp_sum(mine);
  if ((threadIdx.x & 31) == 0) atomicAdd(&s_cnt, mine);
  __syncthreads();
  if (threadIdx.x == 0) tile_counts[blockIdx.x] = (uint32_t)s_cnt;
}

// one CTA: exclusive scan of the tile counts in place, total -> header
__global__ void __launch_bounds__(1024) compact_scan_kernel(uint32_t *__restrict__ tile_counts, int n_tiles, uint32_t n_chunks, uint32_t budget_chunks,
                                                           uint32_t *__restrict__ header)
{
  __shared__ uint32_t s_part[1024];
  const int per = (n_tiles + 1023) / 1024;
  uint32_t local = 0;
  for (int k = 0; k < per; ++k) { const int i = threadIdx.x * per + k; if (i < n_tiles) local += tile_counts[i]; }
  s_part[threadIdx.x] = local;
  __syncthreads();
  for (int o = 1; o < 1024; o <<= 1) {                       // Hillis-Steele inclusive scan
    const uint32_t v = threadIdx.x >= o ? s_part[threadIdx.x - o] : 0;
    __syncthreads();
    s_part[threadIdx.x] += v;
    __syncthreads();
  }
  uint32_t run = s_part[threadIdx.x] - local;
  for (int k = 0; k < per; ++k) { const int i = threadIdx.x * per + k; if (i < n_tiles) { const uint32_t c = tile_counts[i]; tile_counts[i] = run; run += c; } }
  if (threadIdx.x == 1023) { header[0] = s_part[1023]; header[1] = n_chunks; header[2] = s_part[1023] < budget_chunks ? s_part[1023] : budget_chunks; }
}

__global__ void __launch_bounds__(256) compact_write_kernel(const uint4 *__restrict__ region, uint32_t n_chunks, const uint32_t *__restrict__ tile_offsets,
                                                            uint32_t *__restrict__ bitmap, uint4 *__restrict__ packed)
{
  __shared__ uint32_t s_warp_cnt[CMP_TILE / 32];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  uint32_t masks[CMP_TILE / 256];
#pragma unroll
  for (int k = 0; k < CMP_TILE / 256; ++k) {
    const uint32_t c = blockIdx.x * CMP_TILE + k * 256 + threadIdx.x;
    const bool nz = c < n_chunks && chunk_nonzero(region + 2 * (size_t)c);
    masks[k] = __ballot_sync(0xffffffffu, nz);
    if (lane == 0) {
      s_warp_cnt[k * 8 + warp] = __popc(masks[k]);
      if (blockIdx.x * CMP_TILE + k * 256 + warp * 32 < n_chunks) bitmap[(blockIdx.x * CMP_TILE + k * 256) / 32 + warp] = masks[k];
    }
  }
  __syncthreads();
  const uint32_t base = tile_offsets[blockIdx.x];
#pragma unroll
  for (int k = 0; k < CMP_TILE / 256; ++k) {
    if (!((masks[k] >> lane) & 1)) continue;
    uint32_t before = 0;
    for (int j = 0; j < k * 8 + warp; ++j) before += s_warp_cnt[j];           // chunk order = (k, warp, lane)
    const uint32_t dst = base + before + __popc(masks[k] & ((1u << lane) - 1));
    const uint32_t c = blockIdx.x * CMP_TILE + k * 256 + threadIdx.x;
    packed[2 * (size_t)dst] = region[2 * (size_t)c];
    packed[2 * (size_t)dst + 1] = region[2 * (size_t)c + 1];
  }
}

}  // namespace kvzc

using namespace kvzc;

// inter CU residual coding over a TU grid (used by interpass.cu): src/pred/rec point at the grid's first sample
namespace kvzc {
int launch_recon_inter(const kvz_cuda_quant_params &qp, const uint8_t *src, const uint8_t *pred, int stride, int color, int log2w,
                       int blocks_x, int nblk, uint8_t *rec, int16_t *coeff, int32_t *has, uint32_t *ssd, cudaStream_t st)
{
  const int ww = 1 << (2 * log2w), g = 1024 / ww, grid = (nblk + g - 1) / g;
  uint8_t *h8 = reinterpret_cast<uint8_t *>(has);
  switch (log2w) {
    case 2: intra_recon_kernel<uint8_t, 2, true><<<grid, 256, 0, st>>>(qp, src, pred, stride, 0, 0, color, blocks_x, nblk, nullptr, rec, coeff, h8, ssd); break;
    case 3: intra_recon_kernel<uint8_t, 3, true><<<grid, 256, 0, st>>>(qp, src, pred, stride, 0, 0, color, blocks_x, nblk, nullptr, rec, coeff, h8, ssd); break;
    case 4: intra_recon_kernel<uint8_t, 4, true><<<grid, 256, 0, st>>>(qp, src, pred, stride, 0, 0, color, blocks_x, nblk, nullptr, rec, coeff, h8, ssd); break;
    default: intra_recon_kernel<uint8_t, 5, true><<<grid, 256, 0, st>>>(qp, src, pred, stride, 0, 0, color, blocks_x, nblk, nullptr, rec, coeff, h8, ssd); break;
  }
  KVZC_LAUNCHED();
  return 0;
}
}  // namespace kvzc

template <int PHASE, class T>
static int launch_recon_phase(const kvz_cuda_quant_params &qp, const T *src, const T *rin, int stride, int pic_w, int pic_h,
                              int color, int log2w, int blocks_x, int nblk, const int8_t *modes, T *rec, int16_t *coeff,
                              uint8_t *has, uint32_t *ssd, cudaStream_t st)
{
  const int ww = 1 << (2 * log2w), g = 1024 / ww, grid = (nblk + g - 1) / g;
  switch (log2w) {
    case 2: intra_recon_kernel<T, 2, false, PHASE><<<grid, 256, 0, st>>>(qp, src, rin, stride, pic_w, pic_h, color, blocks_x, nblk, modes, rec, coeff, has, ssd); break;
    case 3: intra_recon_kernel<T, 3, false, PHASE><<<grid, 256, 0, st>>>(qp, src, rin, stride, pic_w, pic_h, color, blocks_x, nblk, modes, rec, coeff, has, ssd); break;
    case 4: intra_recon_kernel<T, 4, false, PHASE><<<grid, 256, 0, st>>>(qp, src, rin, stride, pic_w, pic_h, color, blocks_x, nblk, modes, rec, coeff, has, ssd); break;
    default: intra_recon_kernel<T, 5, false, PHASE><<<grid, 256, 0, st>>>(qp, src, rin, stride, pic_w, pic_h, color, blocks_x, nblk, modes, rec, coeff, has, ssd); break;
  }
  KVZC_LAUNCHED();
  return 0;
}

// 4x4 luma with transform skip (PHASE 0 fused / 1 forward / 2 inverse)
template <int PHASE, class T>
static int launch_recon_trskip(const kvz_cuda_quant_params &qp, const T *src, const T *rin, int stride, int pic_w, int pic_h,
                               int blocks_x, int nblk, const int8_t *modes, T *rec, int16_t *coeff, uint8_t *has, uint32_t *ssd, cudaStream_t st)
{
  intra_recon_kernel<T, 2, false, PHASE, true><<<(nblk + 63) / 64, 256, 0, st>>>(qp, src, rin, stride, pic_w, pic_h, 0, blocks_x, nblk, modes, rec, coeff, has, ssd);
  KVZC_LAUNCHED();
  return 0;
}

// kvz_quantize_residual_trskip's decision per 4x4 luma TU (transform.c:241-288): keep the DST result unless the
// transform-skip result has the strictly smaller  SSD + bits * lambda; the winner's data replaces the main sections.
template <class T>
__global__ void __launch_bounds__(256) trskip_select_kernel(int nblk, int blocks_x, int stride, double lambda, const uint32_t *__restrict__ ssd_ts,
                                                            const double *__restrict__ bits_ts, const uint8_t *__restrict__ has_ts,
                                                            const int16_t *__restrict__ coeff_ts, const T *__restrict__ rec_ts,
                                                            uint32_t *__restrict__ ssd, double *__restrict__ bits, uint8_t *__restrict__ has,
                                                            int16_t *__restrict__ coeff, T *__restrict__ rec, uint8_t *__restrict__ flag)
{
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= nblk) return;
  const double cost_ns = (double)ssd[b] + bits[b] * lambda;
  const double cost_ts = (double)ssd_ts[b] + bits_ts[b] * lambda;
  const bool use_ts = !(cost_ns <= cost_ts);
  flag[b] = use_ts;
  if (!use_ts) return;
  ssd[b] = ssd_ts[b]; bits[b] = bits_ts[b]; has[b] = has_ts[b];
  const uint4 *cs = reinterpret_cast<const uint4 *>(coeff_ts + (size_t)b * 16);
  uint4 *cd = reinterpret_cast<uint4 *>(coeff + (size_t)b * 16);
  cd[0] = cs[0]; cd[1] = cs[1];
  const long o = (long)((b / blocks_x) * 4) * stride + (b % blocks_x) * 4;
  for (int y = 0; y < 4; ++y)
    for (int x = 0; x < 4; ++x) rec[o + (long)y * stride + x] = rec_ts[o + (long)y * stride + x];
}

template <class T>
static int launch_recon(const kvz_cuda_quant_params &qp, const T *src, const T *rin, int stride, int pic_w, int pic_h,
                        int color, int log2w, int blocks_x, int nblk, const int8_t *modes, T *rec, int16_t *coeff,
                        uint8_t *has, uint32_t *ssd, cudaStream_t st)
{
  const int ww = 1 << (2 * log2w), g = 1024 / ww, grid = (nblk + g - 1) / g;
  switch (log2w) {
    case 2: intra_recon_kernel<T, 2><<<grid, 256, 0, st>>>(qp, src, rin, stride, pic_w, pic_h, color, blocks_x, nblk, modes, rec, coeff, has, ssd); break;
    case 3: intra_recon_kernel<T, 3><<<grid, 256, 0, st>>>(qp, src, rin, stride, pic_w, pic_h, color, blocks_x, nblk, modes, rec, coeff, has, ssd); break;
    case 4: intra_recon_kernel<T, 4><<<grid, 256, 0, st>>>(qp, src, rin, stride, pic_w, pic_h, color, blocks_x, nblk, modes, rec, coeff, has, ssd); break;
    default: intra_recon_kernel<T, 5><<<grid, 256, 0, st>>>(qp, src, rin, stride, pic_w, pic_h, color, blocks_x, nblk, modes, rec, coeff, has, ssd); break;
  }
  KVZC_LAUNCHED();
  return 0;
}

struct Section { size_t off, bytes; };

struct kvz_cuda_frame_pass {
  kvz_cuda_fp_params prm;
  int W, H;
  int nblk[4], wl[4];
  int nctu3;
  kvz_cuda_fp_layout lay;
  size_t host_bytes, total_bytes;
  uint8_t *blob = nullptr;              // device: host-visible sections first, device-only sections after
  // device-only
  size_t off_rec_y[4], off_rec_u[3], off_rec_v[3];
  size_t off_sao_off, off_dbk_cus, off_cabac, off_src_copy, off_compact, off_tile_counts;
  size_t off_ts_rec = 0, off_ts_coeff = 0, off_ts_has = 0, off_ts_ssd = 0, off_ts_bits = 0;
  kvz_cuda_rdoq_params rdoq;
  std::vector<uint8_t> host_init;       // initial content of the descriptor sections
  size_t init_off = 0, init_bytes = 0;
  // optional per-stage CUDA-event timing (bench.py's live roofline measurement)
  bool timing = false;
  cudaEvent_t ev[KVZ_CUDA_FP_STAGES + 1] = {};
  double ms_acc[KVZ_CUDA_FP_STAGES] = {};
  int runs_timed = 0;
  bool ev_pending = false;
};

// transform-depth below the CU that the pass assumes per quadtree depth index (32x32 TU inside a 64x64 CU, 4x4 = NxN
// split of an 8x8 CU); it only selects the cbf context of RDOQ (rdo.c:895-899).  The CPU arm uses the same table.
static const int k_fp_tr_depth[4] = { 1, 0, 0, 1 };

static void fp_mark(kvz_cuda_frame_pass *fp, int idx, cudaStream_t st) { if (fp->timing) cudaEventRecord(fp->ev[idx], st); }
static void fp_collect(kvz_cuda_frame_pass *fp)
{
  if (!fp->ev_pending) return;
  cudaEventSynchronize(fp->ev[KVZ_CUDA_FP_STAGES]);
  for (int i = 0; i < KVZ_CUDA_FP_STAGES; ++i) { float ms = 0; cudaEventElapsedTime(&ms, fp->ev[i], fp->ev[i + 1]); fp->ms_acc[i] += ms; }
  fp->runs_timed++;
  fp->ev_pending = false;
}

static size_t align_up(size_t v) { return (v + 255) & ~size_t(255); }

extern "C" {

static kvz_cuda_frame_pass *fp_build(const kvz_cuda_fp_params *p, bool alloc)
{
  if (alloc && g_device < 0 && kvz_cuda_init(-1) != 0) return nullptr;
  if (!p || (p->bitdepth != 8 && p->bitdepth != 10) || p->width % 8 || p->height % 8 || p->width < 64 || p->height < 64) {
    set_error("frame pass: need 8- or 10-bit, width/height multiples of 8 and >= 64");
    return nullptr;
  }
  const size_t px = p->bitdepth == 8 ? 1 : 2;            // bytes per sample (kvz_pixel)
  kvz_cuda_frame_pass *fp = new kvz_cuda_frame_pass();
  fp->prm = *p;
  const int W = fp->W = p->width, H = fp->H = p->height;
  size_t off = 0;
  auto take = [&](size_t bytes) { size_t o = off; off = align_up(off + bytes); return o; };
  kvz_cuda_fp_layout &L = fp->lay;
  memset(&L, 0, sizeof(L));
  for (int d = 0; d < 4; ++d) {
    const int w = fp->wl[d] = 32 >> d;
    const int nb = fp->nblk[d] = (W / w) * (H / w);
    L.nblk[d] = nb;
    L.mode_y[d] = take(nb); L.cost_y[d] = take(4 * (size_t)nb); L.has_y[d] = take(nb); L.ssd_y[d] = take(4 * (size_t)nb);
    L.bits_y[d] = take(8 * (size_t)nb);
    if (d == 3) L.trskip_y = take(nb);
    if (d < 3) {
      L.has_u[d] = take(nb); L.has_v[d] = take(nb); L.ssd_u[d] = take(4 * (size_t)nb); L.ssd_v[d] = take(4 * (size_t)nb);
      L.bits_u[d] = take(8 * (size_t)nb); L.bits_v[d] = take(8 * (size_t)nb);
    }
  }
  const int cx = (W + 63) / 64, cy = (H + 63) / 64, nctu = cx * cy;
  fp->nctu3 = nctu * 3;
  L.nctu = nctu;
  L.sao_stats = take(4 * (size_t)fp->nctu3 * 40); L.sao_dd = take(4 * (size_t)fp->nctu3 * 4);
  L.sao_band_dd = take(4 * (size_t)fp->nctu3); L.sao_best = take(fp->nctu3);
  L.sao_rec = take((size_t)W * H * 3 / 2 * px);
  L.checksum = take(16);
  // the (large, sparse) coefficient sections come last so that the compact result is two copies: the head + the packed chunks
  L.coeff_begin = off;
  for (int d = 0; d < 4; ++d) {
    const int w = fp->wl[d], nb = fp->nblk[d];
    L.coeff_y[d] = take(2 * (size_t)nb * w * w);
    if (d < 3) { const int wc = w / 2; L.coeff_u[d] = take(2 * (size_t)nb * wc * wc); L.coeff_v[d] = take(2 * (size_t)nb * wc * wc); }
  }
  L.host_bytes = fp->host_bytes = off;
  L.n_chunks = (L.host_bytes - L.coeff_begin) / 32;
  L.compact_header_bytes = 256 + align_up((size_t)(L.n_chunks + 7) / 8);
  if (p->trskip) {            // scratch of the transform-skip candidate of every 4x4 luma TU
    const size_t nb3 = fp->nblk[3];
    fp->off_ts_rec = take((size_t)W * H * px); fp->off_ts_coeff = take(2 * nb3 * 16); fp->off_ts_has = take(nb3);
    fp->off_ts_ssd = take(4 * nb3); fp->off_ts_bits = take(8 * nb3);
  }
  fp->off_compact = take(L.compact_header_bytes + (size_t)L.n_chunks * 32);
  fp->off_tile_counts = take(4 * ((size_t)L.n_chunks / 1024 + 2));
  for (int d = 0; d < 4; ++d) fp->off_rec_y[d] = take((size_t)W * H * px);
  for (int d = 0; d < 3; ++d) { fp->off_rec_u[d] = take((size_t)W * H / 4 * px); fp->off_rec_v[d] = take((size_t)W * H / 4 * px); }
  fp->off_sao_off = take(4 * (size_t)4 * fp->nctu3 * 5);
  fp->off_src_copy = take((size_t)W * H * 3 / 2 * px);
  // deblocking input: the CU records of the uniform 8x8 intra quadtree whose reconstruction SAO works on
  // (cu_info_t image: type = CU_INTRA, depth = 3, part_size = 2Nx2N, tr_depth = 3), initialised from the host once
  fp->init_off = off;
  fp->off_dbk_cus = take((size_t)(W / 4) * (H / 4) * 20);
  fp->off_cabac = take(sizeof(kvz_cuda_cabac_ctx));      // slice-initial context models for RDOQ (I slice)
  fp->init_bytes = off - fp->init_off;
  fp->total_bytes = off;
  if (alloc) {
    fp->host_init.assign(fp->init_bytes, 0);
    uint8_t *rec = fp->host_init.data() + (fp->off_dbk_cus - fp->init_off);
    for (size_t i = 0; i < (size_t)(W / 4) * (H / 4); ++i) {
      rec[20 * i + 0] = (uint8_t)(1 | (3 << 2));
      rec[20 * i + 1] = 3;
      rec[20 * i + 6] = (uint8_t)p->qp;
    }
    if (kvz_cuda_cabac_ctx_init(p->qp, 2, (kvz_cuda_cabac_ctx *)(fp->host_init.data() + (fp->off_cabac - fp->init_off))) != 0) { delete fp; return nullptr; }
  }
  fp->rdoq.lambda = p->lambda > 0 ? p->lambda : 0.57 * pow(2.0, (p->qp - 12) / 3.0);
  fp->rdoq.qp = p->qp; fp->rdoq.bitdepth = p->bitdepth; fp->rdoq.signhide_enable = p->signhide; fp->rdoq.pad = 0;
  if (!alloc) return fp;
  if (cudaMalloc((void **)&fp->blob, fp->total_bytes) != cudaSuccess) { set_error("frame pass: cudaMalloc(%zu) failed", fp->total_bytes); delete fp; return nullptr; }
  cudaMemset(fp->blob, 0, fp->total_bytes);
  cudaMemcpy(fp->blob + fp->init_off, fp->host_init.data(), fp->init_bytes, cudaMemcpyHostToDevice);
  return fp;
}

kvz_cuda_frame_pass *kvz_cuda_fp_create(const kvz_cuda_fp_params *p) { return fp_build(p, true); }

/* layout only: needs no device (used by the CPU reference arm and the tests) */
int kvz_cuda_fp_layout_for(const kvz_cuda_fp_params *p, kvz_cuda_fp_layout *out)
{
  KVZC_ARG(out != nullptr);
  kvz_cuda_frame_pass *fp = fp_build(p, false);
  if (!fp) return KVZ_CUDA_E_ARG;
  *out = fp->lay;
  delete fp;
  return 0;
}

void kvz_cuda_fp_destroy(kvz_cuda_frame_pass *fp)
{
  if (!fp) return;
  for (cudaEvent_t ev : fp->ev) if (ev) cudaEventDestroy(ev);
  cudaFree(fp->blob);
  delete fp;
}

int kvz_cuda_fp_layout_get(const kvz_cuda_frame_pass *fp, kvz_cuda_fp_layout *out) { KVZC_ARG(fp && out); *out = fp->lay; return 0; }
void *kvz_cuda_fp_result_dev(kvz_cuda_frame_pass *fp) { return fp ? fp->blob : nullptr; }
size_t kvz_cuda_fp_frame_bytes(const kvz_cuda_frame_pass *fp) { return fp ? (size_t)fp->W * fp->H * 3 / 2 * (fp->prm.bitdepth == 8 ? 1 : 2) : 0; }

}  // extern "C"

template <class T>
static int fp_run_dev_t(kvz_cuda_frame_pass *fp, const void *src_dev, const void *rec_in_dev, cudaStream_t st)
{
  constexpr int BD = PixTraits<T>::bd;
  const int W = fp->W, H = fp->H;
  const T *src = (const T *)src_dev;
  const T *rin = rec_in_dev ? (const T *)rec_in_dev : src;
  uint8_t *B = fp->blob;
  const kvz_cuda_fp_layout &L = fp->lay;
  kvz_cuda_quant_params qp = { fp->prm.qp, BD, 1, fp->prm.signhide, 0 };
  const size_t poff[3] = { 0, (size_t)W * H, (size_t)W * H * 5 / 4 };
  if (fp->timing) fp_collect(fp);
  const bool rdoq = fp->prm.rdoq != 0;
  const kvz_cuda_cabac_ctx *cabac = (const kvz_cuda_cabac_ctx *)(B + fp->off_cabac);
  for (int d = 0; d < 4; ++d) {
    const int w = fp->wl[d], log2w = 5 - d, nb = fp->nblk[d];
    const int s0 = d * 9;                 // stage slots: rough, luma fwd (or fused), luma rdoq, luma inv, luma bits, chroma fwd, rdoq, inv, bits
    fp_mark(fp, s0 + 0, st);
    if (nb == 0) { for (int k = 1; k < 9; ++k) fp_mark(fp, s0 + k, st); continue; }
    int8_t *modes = (int8_t *)(B + L.mode_y[d]);
    // rough search with the mode selection fused in; the 35-entry cost tables stay on chip
    if constexpr (BD == 8) {
      if (int r = rough_search_u8(log2w, src, rin, W, W, H, nullptr, modes, (uint32_t *)(B + L.cost_y[d]), st)) return r;
    } else {
      if (int r = rough_search_u16(log2w, src, rin, W, W, H, nullptr, modes, (uint32_t *)(B + L.cost_y[d]), st)) return r;
    }
    fp_mark(fp, s0 + 1, st);
    // luma: prediction -> transform -> quantisation -> reconstruction; with RDOQ the fused kernel is split around the
    // RDOQ launch (quant-generic.c:234-240)
    {
      T *rec = (T *)(B + fp->off_rec_y[d]);
      uint8_t *has = B + L.has_y[d];
      int16_t *coeff = (int16_t *)(B + L.coeff_y[d]);
      uint32_t *ssd = (uint32_t *)(B + L.ssd_y[d]);
      if (!rdoq) {
        if (int r = launch_recon(qp, src, rin, W, W, H, 0, log2w, W / w, nb, modes, rec, coeff, has, ssd, st)) return r;
        fp_mark(fp, s0 + 2, st); fp_mark(fp, s0 + 3, st);
      } else {
        if (int r = launch_recon_phase<1>(qp, src, rin, W, W, H, 0, log2w, W / w, nb, modes, rec, coeff, has, ssd, st)) return r;
        fp_mark(fp, s0 + 2, st);
        if (int r = rdoq_launch_grid(fp->rdoq, cabac, coeff, nullptr, nb, log2w, modes, 0, k_fp_tr_depth[d], st)) return r;
        fp_mark(fp, s0 + 3, st);
        if (int r = launch_recon_phase<2>(qp, src, rin, W, W, H, 0, log2w, W / w, nb, modes, rec, coeff, has, ssd, st)) return r;
      }
    }
    fp_mark(fp, s0 + 4, st);
    // CABAC bit cost of the luma levels (kvz_get_coeff_cost, rdo.c:291-330) with the slice-initial context models
    const int ts_flag = (d == 3 && fp->prm.trskip) ? 1 : 0;              // 4x4 TUs: the transform_skip_flag bin is part of the count
    if (int r = coeff_cost_launch_grid(fp->prm.signhide, cabac, (const int16_t *)(B + L.coeff_y[d]), nullptr, nb, log2w, modes, ts_flag, (double *)(B + L.bits_y[d]), nullptr, st)) return r;
    if (ts_flag) {
      // the transform-skip candidate of every 4x4 luma TU, then kvz_quantize_residual_trskip's choice (stage slot: luma bits)
      T *rec_ts = (T *)(B + fp->off_ts_rec);
      uint8_t *has_ts = B + fp->off_ts_has;
      int16_t *coeff_ts = (int16_t *)(B + fp->off_ts_coeff);
      uint32_t *ssd_ts = (uint32_t *)(B + fp->off_ts_ssd);
      double *bits_ts = (double *)(B + fp->off_ts_bits);
      if (!rdoq) {
        if (int r = launch_recon_trskip<0>(qp, src, rin, W, W, H, W / w, nb, modes, rec_ts, coeff_ts, has_ts, ssd_ts, st)) return r;
      } else {
        if (int r = launch_recon_trskip<1>(qp, src, rin, W, W, H, W / w, nb, modes, rec_ts, coeff_ts, has_ts, ssd_ts, st)) return r;
        if (int r = rdoq_launch_grid(fp->rdoq, cabac, coeff_ts, nullptr, nb, log2w, modes, 0, k_fp_tr_depth[d], st)) return r;
        if (int r = launch_recon_trskip<2>(qp, src, rin, W, W, H, W / w, nb, modes, rec_ts, coeff_ts, has_ts, ssd_ts, st)) return r;
      }
      if (int r = coeff_cost_launch_grid(fp->prm.signhide, cabac, coeff_ts, nullptr, nb, log2w, modes, 1, bits_ts, nullptr, st)) return r;
      trskip_select_kernel<T><<<(nb + 255) / 256, 256, 0, st>>>(nb, W / w, W, fp->rdoq.lambda, ssd_ts, bits_ts, has_ts, coeff_ts, rec_ts,
                                                             (uint32_t *)(B + L.ssd_y[d]), (double *)(B + L.bits_y[d]), B + L.has_y[d],
                                                             (int16_t *)(B + L.coeff_y[d]), (T *)(B + fp->off_rec_y[d]), B + L.trskip_y);
      KVZC_LAUNCHED();
    }
    fp_mark(fp, s0 + 5, st);
    if (d == 3) { fp_mark(fp, s0 + 6, st); fp_mark(fp, s0 + 7, st); fp_mark(fp, s0 + 8, st); continue; }
    const int wc = w / 2;
    for (int step = 0; step < 4; ++step) {
      // RDOQ and the bit cost take U and V in ONE launch (twice the TUs in flight for these latency-bound kernels)
      if (step == 1 && rdoq) {
        if (int r = rdoq_launch_grid(fp->rdoq, cabac, (int16_t *)(B + L.coeff_u[d]), (int16_t *)(B + L.coeff_v[d]), nb, log2w - 1, modes, 1, k_fp_tr_depth[d], st)) return r;
      } else if (step == 3) {
        if (int r = coeff_cost_launch_grid(fp->prm.signhide, cabac, (const int16_t *)(B + L.coeff_u[d]), (const int16_t *)(B + L.coeff_v[d]), nb, log2w - 1,
                                           modes, fp->prm.trskip /* counted for 4x4 chroma TUs too */, (double *)(B + L.bits_u[d]), (double *)(B + L.bits_v[d]), st, 1)) return r;
      } else
      for (int color = 1; color <= 2 && (rdoq || step == 0); ++color) {
        const T *csrc = src + poff[color], *crin = rin + poff[color];
        T *rec = (T *)(B + (color == 1 ? fp->off_rec_u[d] : fp->off_rec_v[d]));
        uint8_t *has = B + (color == 1 ? L.has_u[d] : L.has_v[d]);
        int16_t *coeff = (int16_t *)(B + (color == 1 ? L.coeff_u[d] : L.coeff_v[d]));
        uint32_t *ssd = (uint32_t *)(B + (color == 1 ? L.ssd_u[d] : L.ssd_v[d]));
        int r = 0;
        if (!rdoq) r = launch_recon(qp, csrc, crin, W / 2, W, H, color, log2w - 1, (W / 2) / wc, nb, modes, rec, coeff, has, ssd, st);
        else if (step == 0) r = launch_recon_phase<1>(qp, csrc, crin, W / 2, W, H, color, log2w - 1, (W / 2) / wc, nb, modes, rec, coeff, has, ssd, st);
        else r = launch_recon_phase<2>(qp, csrc, crin, W / 2, W, H, color, log2w - 1, (W / 2) / wc, nb, modes, rec, coeff, has, ssd, st);
        if (r) return r;
      }
      if (step < 3) fp_mark(fp, s0 + 6 + step, st);
    }
  }
  fp_mark(fp, 36, st);
  // ---- deblocking of the 8x8-level reconstruction (depth index 2) in place: every 8x8 edge is an intra TU edge ----
  {
    kvz_cuda_dbk_params dp;
    memset(&dp, 0, sizeof(dp));
    dp.width = W; dp.height = H; dp.qp = fp->prm.qp; dp.cu_stride_scu = W / 4;
    if (int r = kvz_cuda_deblock_frame(&dp, BD, B + fp->off_rec_y[2], B + fp->off_rec_u[2], B + fp->off_rec_v[2], B + fp->off_dbk_cus, st)) return r;
  }
  fp_mark(fp, 37, st);
  // ---- SAO on the deblocked reconstruction: statistics + decisions, then reconstruction ----
  const int nctu = fp->nctu3 / 3;
  SaoPlanesT<T> pl;
  for (int color = 0; color < 3; ++color) {
    pl.src[color] = src + poff[color];
    pl.rec[color] = (const T *)(B + (color == 0 ? fp->off_rec_y[2] : (color == 1 ? fp->off_rec_u[2] : fp->off_rec_v[2])));
    pl.out[color] = (T *)(B + L.sao_rec) + poff[color];
    pl.Wp[color] = color ? W / 2 : W; pl.Hp[color] = color ? H / 2 : H;
  }
  int32_t *dec_off = (int32_t *)(B + fp->off_sao_off);
  uint32_t *ck_scratch = (uint32_t *)(B + fp->off_sao_off) + (size_t)fp->nctu3 * 5;
  sao_ctu_kernel<<<fp->nctu3, 256, 0, st>>>(pl, nctu, (W + 63) / 64, (int32_t *)(B + L.sao_stats), (int32_t *)(B + L.sao_dd),
                                            (int32_t *)(B + L.sao_band_dd), (int8_t *)(B + L.sao_best), dec_off, ck_scratch);
  KVZC_LAUNCHED();
  fp_mark(fp, 38, st);
  sao_apply_kernel<<<fp->nctu3, 256, 0, st>>>(pl, nctu, (W + 63) / 64, (const int8_t *)(B + L.sao_best), dec_off);
  KVZC_LAUNCHED();
  fp_mark(fp, 39, st);
  // ---- picture checksum of the filtered planes ----
  if constexpr (BD == 8) {
    checksum3_kernel<<<dim3(g_sm_count, 3), 256, 0, st>>>(pl, ck_scratch, B + L.checksum);
    KVZC_LAUNCHED();
  } else {
    for (int color = 0; color < 3; ++color)
      if (int r = kvz_cuda_array_checksum(BD, pl.out[color], pl.Hp[color], pl.Wp[color], pl.Wp[color], B + L.checksum + 4 * color, st)) return r;
  }
  fp_mark(fp, KVZ_CUDA_FP_STAGES, st);
  if (fp->timing) fp->ev_pending = true;
  return 0;
}

extern "C" {

int kvz_cuda_fp_run_dev(kvz_cuda_frame_pass *fp, const void *src_dev, const void *rec_in_dev, void *stream)
{
  KVZC_REQUIRE_DEVICE();
  KVZC_ARG(fp && src_dev);
  if (fp->prm.bitdepth == 8) return fp_run_dev_t<uint8_t>(fp, src_dev, rec_in_dev, as_stream(stream));
  return fp_run_dev_t<uint16_t>(fp, src_dev, rec_in_dev, as_stream(stream));
}

int kvz_cuda_fp_set_timing(kvz_cuda_frame_pass *fp, int enable)
{
  KVZC_ARG(fp != nullptr);
  if (enable && !fp->ev[0]) for (int i = 0; i <= KVZ_CUDA_FP_STAGES; ++i) KVZC_CHECK(cudaEventCreate(&fp->ev[i]));
  fp->timing = enable != 0;
  fp->ev_pending = false;
  fp->runs_timed = 0;
  for (int i = 0; i < KVZ_CUDA_FP_STAGES; ++i) fp->ms_acc[i] = 0;
  return 0;
}

int kvz_cuda_fp_get_timing(kvz_cuda_frame_pass *fp, double *ms_total, int *runs)
{
  KVZC_ARG(fp && ms_total && runs);
  fp_collect(fp);
  for (int i = 0; i < KVZ_CUDA_FP_STAGES; ++i) ms_total[i] = fp->ms_acc[i];
  *runs = fp->runs_timed;
  return 0;
}

int kvz_cuda_fp_run_host_compact(kvz_cuda_frame_pass *fp, const void *src_host, void *small_host, void *compact_host, uint32_t budget_chunks,
                                 void *stream)
{
  KVZC_REQUIRE_DEVICE();
  KVZC_ARG(fp && src_host && small_host && compact_host);
  cudaStream_t st = as_stream(stream);
  const kvz_cuda_fp_layout &L = fp->lay;
  uint8_t *B = fp->blob;
  uint8_t *src_dev = B + fp->off_src_copy;
  KVZC_CHECK(cudaMemcpyAsync(src_dev, src_host, kvz_cuda_fp_frame_bytes(fp), cudaMemcpyHostToDevice, st));
  if (int r = kvz_cuda_fp_run_dev(fp, src_dev, nullptr, st)) return r;
  const uint32_t n_chunks = (uint32_t)L.n_chunks, n_tiles = (n_chunks + CMP_TILE - 1) / CMP_TILE;
  uint8_t *cmp = B + fp->off_compact;
  uint32_t *tiles = (uint32_t *)(B + fp->off_tile_counts);
  const uint4 *region = (const uint4 *)(B + L.coeff_begin);
  compact_count_kernel<<<n_tiles, 256, 0, st>>>(region, n_chunks, tiles);
  KVZC_LAUNCHED();
  if (budget_chunks > n_chunks) budget_chunks = n_chunks;
  compact_scan_kernel<<<1, 1024, 0, st>>>(tiles, (int)n_tiles, n_chunks, (uint32_t)budget_chunks, (uint32_t *)cmp);
  KVZC_LAUNCHED();
  compact_write_kernel<<<n_tiles, 256, 0, st>>>(region, n_chunks, tiles, (uint32_t *)(cmp + 256), (uint4 *)(cmp + L.compact_header_bytes));
  KVZC_LAUNCHED();
  KVZC_CHECK(cudaMemcpyAsync(small_host, B, L.coeff_begin, cudaMemcpyDeviceToHost, st));
  KVZC_CHECK(cudaMemcpyAsync(compact_host, cmp, L.compact_header_bytes + (size_t)budget_chunks * 32, cudaMemcpyDeviceToHost, st));
  return 0;
}

int kvz_cuda_fp_expand_compact(const kvz_cuda_fp_layout *layout, const void *compact_host, size_t compact_bytes, void *coeff_region_out)
{
  KVZC_ARG(layout && compact_host && coeff_region_out && compact_bytes >= layout->compact_header_bytes);
  const uint8_t *c = (const uint8_t *)compact_host;
  uint32_t head[2];
  memcpy(head, c, sizeof(head));
  const uint64_t n_chunks = layout->n_chunks;
  KVZC_ARG(head[1] == n_chunks);
  KVZC_ARG((compact_bytes - layout->compact_header_bytes) / 32 >= head[0]);
  const uint32_t *bitmap = (const uint32_t *)(c + 256);
  const uint8_t *packed = c + layout->compact_header_bytes;
  uint8_t *out = (uint8_t *)coeff_region_out;
  memset(out, 0, (size_t)n_chunks * 32);
  uint64_t src = 0;
  for (uint64_t w = 0; w < (n_chunks + 31) / 32; ++w) {
    uint32_t m = bitmap[w];
    while (m) {
      const int b = __builtin_ctz(m);
      m &= m - 1;
      memcpy(out + (w * 32 + b) * 32, packed + src * 32, 32);
      ++src;
    }
  }
  KVZC_ARG(src == head[0]);
  return 0;
}

int kvz_cuda_fp_compact_fetch(kvz_cuda_frame_pass *fp, uint32_t first_chunk, uint32_t count, void *dst_host, void *stream)
{
  KVZC_REQUIRE_DEVICE();
  KVZC_ARG(fp && dst_host && (uint64_t)first_chunk + count <= fp->lay.n_chunks);
  KVZC_CHECK(cudaMemcpyAsync(dst_host, fp->blob + fp->off_compact + fp->lay.compact_header_bytes + (size_t)first_chunk * 32, (size_t)count * 32,
                             cudaMemcpyDeviceToHost, as_stream(stream)));
  return 0;
}

int kvz_cuda_fp_run_host(kvz_cuda_frame_pass *fp, const void *src_host, void *result_host, void *stream)
{
  KVZC_REQUIRE_DEVICE();
  KVZC_ARG(fp && src_host && result_host);
  cudaStream_t st = as_stream(stream);
  uint8_t *src_dev = fp->blob + fp->off_src_copy;
  KVZC_CHECK(cudaMemcpyAsync(src_dev, src_host, kvz_cuda_fp_frame_bytes(fp), cudaMemcpyHostToDevice, st));
  if (int r = kvz_cuda_fp_run_dev(fp, src_dev, nullptr, st)) return r;
  KVZC_CHECK(cudaMemcpyAsync(result_host, fp->blob, fp->host_bytes, cudaMemcpyDeviceToHost, st));
  return 0;
}

}  // extern "C"
