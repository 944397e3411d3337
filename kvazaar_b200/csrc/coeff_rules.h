// coeff_rules.h -- the reference's coefficient-coding rules, written once for every device path that quantises or
// counts coefficients: the strategy kernels (namespace kvzc), the CTU search driver (namespace kvzctu) and its host
// builds (g++, one-thread CTA).  Nothing here depends on where a caller keeps its tables or how many threads walk a
// unit: the walks that differ in that respect pass what they differ in (a table pointer, a policy object).
//
//   * tables: entropy bits, CABAC state transitions, quantiser scales, the 4x4 significance map, min_in_group -- as
//     macro lists, expanded into host arrays (ctu_tables_init) and device arrays (the strategy kernels);
//   * scalar rules: kvz_get_scaled_qp, the scan order of a block of up to 8x8, the last-position group index;
//   * context-model offsets into the kvz_cuda_cabac_ctx image;
//   * RDOQ: level rate, significance context, sign hiding; kvz_quant's sign hiding;
//   * the CABAC bit count of a transform unit (kvz_get_coeff_cost's CABAC branch).
#pragma once
#include <stdint.h>
#include <stddef.h>
#include "../../include/kvz_cuda.h"

#if defined(__CUDACC__)
#define COEFF_FN __device__ __forceinline__                 // rules only device code evaluates
#define COEFF_HD __host__ __device__ __forceinline__        // rules the host also evaluates (table construction)
#define COEFF_MFN __device__ __forceinline__                // member functions of policies
#else
#define COEFF_FN static inline
#define COEFF_HD static inline
#define COEFF_MFN inline
#endif

// ---------------------------------------------------------------------------------------------- tables
// HM's fractional-bit estimates per CABAC state, 15 fractional bits, by symbol = MPS / LPS (kvz_entropy_bits,
// rdo.c:69-79: entry [2s] is the MPS cost of state s, [2s + 1] the LPS cost)
#define COEFF_EBITS_MPS \
  32768, 30426, 28306, 26378, 24617, 23005, 21523, 20159, 18899, 17734, 16653, 15650, 14717, 13849, 13038, 12282, \
  11575, 10914, 10294, 9714, 9169, 8658, 8178, 7727, 7303, 6903, 6527, 6173, 5840, 5525, 5228, 4948, \
  4684, 4435, 4199, 3977, 3767, 3568, 3380, 3202, 3034, 2876, 2725, 2583, 2448, 2321, 2200, 2086, \
  1978, 1875, 1778, 1686, 1599, 1517, 1439, 1364, 1294, 1228, 1165, 1105, 1048, 994, 943, 895
#define COEFF_EBITS_LPS \
  32768, 35232, 37696, 40159, 42623, 45087, 47551, 50015, 52479, 54942, 57406, 59870, 62334, 64798, 67262, 69725, \
  72189, 74653, 77117, 79581, 82044, 84508, 86972, 89436, 91900, 94363, 96827, 99291, 101755, 104219, 106683, 109146, \
  111610, 114074, 116538, 119002, 121465, 123929, 126393, 128857, 131321, 133785, 136248, 138712, 141176, 143640, 146104, 148568, \
  151031, 153495, 155959, 158423, 160887, 163351, 165814, 168278, 170742, 173207, 175669, 178134, 180598, 183061, 185525, 187989
// next pStateIdx after an LPS (table 9-41 of the standard; kvz_g_auc_next_state_lps, cabac.c:40-62)
#define COEFF_TRANS_LPS \
  0, 0, 1, 2, 2, 4, 4, 5, 6, 7, 8, 9, 9, 11, 11, 12, 13, 13, 15, 15, 16, 16, 18, 18, 19, 19, 21, 21, 22, 22, 23, 24, \
  24, 25, 26, 26, 27, 27, 28, 29, 29, 30, 30, 30, 31, 32, 32, 33, 33, 33, 34, 34, 35, 35, 35, 36, 36, 36, 37, 37, 37, 38, 38, 63
#define COEFF_QUANT_SCALES 26214, 23302, 20560, 18396, 16384, 14564       // scalinglist.c:78
#define COEFF_INV_QUANT_SCALES 40, 45, 51, 57, 64, 72                     // scalinglist.c:79
#define COEFF_SIG_CTX4 0, 1, 4, 5, 2, 3, 4, 5, 6, 6, 8, 8, 7, 7, 8, 8     // ctx_ind_map of 4x4 blocks (context.c:366)
#define COEFF_MIN_IN_GROUP 0, 1, 2, 3, 4, 6, 8, 12, 16, 24                // g_min_in_group

namespace kvzcoeff {

constexpr int RDOQ_ONE_BIT = 1 << 15;

COEFF_HD int imin(int a, int b) { return a < b ? a : b; }
COEFF_HD int iabs(int a) { return a < 0 ? -a : a; }

// CABAC state transitions on the packed state byte (pStateIdx << 1 | valMps)
COEFF_HD uint8_t cabac_next_mps(int uc) { return (uint8_t)(uc < 124 ? uc + 2 : uc); }
COEFF_HD uint8_t cabac_next_lps(int uc)
{
  const uint8_t trans[64] = { COEFF_TRANS_LPS };
  const int s = uc >> 1, mps = uc & 1;
  return (uint8_t)((trans[s] << 1) | (s == 0 ? 1 - mps : mps));
}

// Six 16-bit table entries packed into two 64-bit immediates, looked up with shifts: a small array indexed at run time
// is built in local memory (the thread's stack) on every use.
struct Pack6x16 { unsigned long long lo, hi; };
COEFF_HD constexpr Pack6x16 pack6x16(int a, int b, int c, int d, int e, int f)
{
  return { (unsigned long long)a | (unsigned long long)b << 16 | (unsigned long long)c << 32 | (unsigned long long)d << 48,
           (unsigned long long)e | (unsigned long long)f << 16 };
}
COEFF_HD int unpack6x16(Pack6x16 p, int r) { return (int)(((r < 4 ? p.lo : p.hi) >> (16 * (r & 3))) & 0xffff); }
COEFF_FN int quant_scale(int r) { constexpr Pack6x16 t = pack6x16(COEFF_QUANT_SCALES); return unpack6x16(t, r); }
COEFF_FN int inv_quant_scale(int r) { constexpr Pack6x16 t = pack6x16(COEFF_INV_QUANT_SCALES); return unpack6x16(t, r); }

// kvz_get_scaled_qp (transform.c:56-62, 88-102) with the chroma QP mapping table folded into its rule; qp_offset is
// the bit depth's 6 * (bitdepth - 8).  type: 0 luma, else chroma.
COEFF_HD int scaled_qp(int type, int qp, int qp_offset)
{
  if (type == 0) return qp + qp_offset;
  int q = qp < -qp_offset ? -qp_offset : (qp > 57 ? 57 : qp);
  if (q < 0) return q + qp_offset;
  int c;
  if (q < 30) c = q;
  else if (q >= 44) c = q - 6;
  else c = q < 34 ? q - 1 : 33 + ((q - 34) >> 1);      // 29, 30, 31, 32, 33, 33, 34, 34, 35, 35, 36, 36, 37, 37
  return c + qp_offset;
}

// raster position of scan index `idx` in a dim x dim block, dim = 1, 2, 4, 8 (kvz_g_sig_last_scan): 0 = up-right
// diagonal, 1 = horizontal, 2 = vertical.  Larger blocks scan their 4x4 groups in this order, and inside each group.
COEFF_HD int scan_small(int scan_idx, int dim_log2, int idx)
{
  const int dim = 1 << dim_log2;
  if (scan_idx == 1) return idx;                                              // (y = idx / dim, x = idx % dim)
  if (scan_idx == 2) return (idx & (dim - 1)) * dim + (idx >> dim_log2);      // x = idx / dim, y = idx % dim
  // diagonal: walk anti-diagonals d = x + y from bottom-left (max y) to top-right
  int d = 0, start = 0;
  for (;; ++d) {
#if defined(__CUDA_ARCH__)
    const int ylo = max(0, d - (dim - 1)), yhi = min(d, dim - 1), len = yhi - ylo + 1;
#else
    const int ylo = d - (dim - 1) > 0 ? d - (dim - 1) : 0, yhi = d < dim - 1 ? d : dim - 1, len = yhi - ylo + 1;
#endif
    if (idx < start + len) { const int y = yhi - (idx - start); return y * dim + (d - y); }
    start += len;
  }
}

// position group of a last-significant coordinate (g_group_idx: 0,1,2,3,4,4,5,5,6,6,6,6,7,7,7,7,8..,9..)
COEFF_HD int last_group(int x)
{
  if (x < 4) return x;
#if defined(__CUDA_ARCH__)
  const int l = 31 - __clz(x);
#else
  const int l = 31 - __builtin_clz(x);
#endif
  return 2 * l + ((x >> (l - 1)) & 1);
}

// ---------------------------------------------------------------------------------------------- context models
// Offsets into the memory image of cabac_data_t.ctx (cabac.h:66-102), which is also kvz_cuda_cabac_ctx.
enum CtxOff {
  CTX_SAO_MERGE = 0, CTX_SAO_TYPE = 1, CTX_SPLIT = 2, CTX_INTRA_MODE = 5, CTX_CHROMA_PRED = 6, CTX_INTER_DIR = 8,
  CTX_TRANS_SUBDIV = 13, CTX_CBF_LUMA = 16, CTX_CBF_CHROMA = 20, CTX_QP_DELTA = 24, CTX_PART_SIZE = 28,
  CTX_SIG_CG = 32, CTX_SIG_LUMA = 36, CTX_SIG_CHROMA = 63, CTX_LAST_Y_LUMA = 78, CTX_LAST_Y_CHROMA = 93,
  CTX_LAST_X_LUMA = 108, CTX_LAST_X_CHROMA = 123, CTX_ONE_LUMA = 138, CTX_ONE_CHROMA = 154, CTX_ABS_LUMA = 162,
  CTX_ABS_CHROMA = 166, CTX_PRED_MODE = 168, CTX_SKIP_FLAG = 169, CTX_MERGE_IDX = 172, CTX_MERGE_FLAG = 173,
  CTX_TQ_BYPASS = 174, CTX_MVD = 175, CTX_REF_PIC = 177, CTX_MVP_IDX = 179, CTX_ROOT_CBF = 181,
  CTX_TRSKIP_LUMA = 182, CTX_TRSKIP_CHROMA = 183, CTX_COUNT = 184
};
#define COEFF_CTX_AT(off, member) static_assert((off) == offsetof(kvz_cuda_cabac_ctx, member), #off)
COEFF_CTX_AT(CTX_SAO_MERGE, sao_merge_flag_model);
COEFF_CTX_AT(CTX_SAO_TYPE, sao_type_idx_model);
COEFF_CTX_AT(CTX_SPLIT, split_flag_model);
COEFF_CTX_AT(CTX_INTRA_MODE, intra_mode_model);
COEFF_CTX_AT(CTX_CHROMA_PRED, chroma_pred_model);
COEFF_CTX_AT(CTX_TRANS_SUBDIV, trans_subdiv_model);
COEFF_CTX_AT(CTX_CBF_LUMA, qt_cbf_model_luma);
COEFF_CTX_AT(CTX_CBF_CHROMA, qt_cbf_model_chroma);
COEFF_CTX_AT(CTX_PART_SIZE, part_size_model);
COEFF_CTX_AT(CTX_SIG_CG, cu_sig_coeff_group_model);
COEFF_CTX_AT(CTX_SIG_LUMA, cu_sig_model_luma);
COEFF_CTX_AT(CTX_SIG_CHROMA, cu_sig_model_chroma);
COEFF_CTX_AT(CTX_LAST_Y_LUMA, cu_ctx_last_y_luma);
COEFF_CTX_AT(CTX_LAST_Y_CHROMA, cu_ctx_last_y_chroma);
COEFF_CTX_AT(CTX_LAST_X_LUMA, cu_ctx_last_x_luma);
COEFF_CTX_AT(CTX_LAST_X_CHROMA, cu_ctx_last_x_chroma);
COEFF_CTX_AT(CTX_ONE_LUMA, cu_one_model_luma);
COEFF_CTX_AT(CTX_ONE_CHROMA, cu_one_model_chroma);
COEFF_CTX_AT(CTX_ABS_LUMA, cu_abs_model_luma);
COEFF_CTX_AT(CTX_ABS_CHROMA, cu_abs_model_chroma);
COEFF_CTX_AT(CTX_ROOT_CBF, cu_qt_root_cbf_model);
COEFF_CTX_AT(CTX_TRSKIP_LUMA, transform_skip_model_luma);
COEFF_CTX_AT(CTX_TRSKIP_CHROMA, transform_skip_model_chroma);
static_assert(CTX_COUNT == sizeof(kvz_cuda_cabac_ctx), "CTX_COUNT");
#undef COEFF_CTX_AT

// ---------------------------------------------------------------------------------------------- RDOQ
struct RdoqModels {      // views into a context-model image for one texture type
  const uint8_t *sig, *one, *abs, *cg, *last_x, *last_y, *cbf;
  const int32_t *eb;     // entropy bits [state byte ^ bin]
  uint8_t root_cbf;
};
COEFF_FN RdoqModels rdoq_models(const uint8_t *cabac, const int32_t *eb, int type)
{
  RdoqModels m;
  m.eb = eb;
  m.sig = cabac + (type ? CTX_SIG_CHROMA : CTX_SIG_LUMA);
  m.one = cabac + (type ? CTX_ONE_CHROMA : CTX_ONE_LUMA);
  m.abs = cabac + (type ? CTX_ABS_CHROMA : CTX_ABS_LUMA);
  m.cg = cabac + CTX_SIG_CG + type;                         // rdo.c:720: indexed by type (0 luma, 2 chroma)
  m.last_x = cabac + (type ? CTX_LAST_X_CHROMA : CTX_LAST_X_LUMA);
  m.last_y = cabac + (type ? CTX_LAST_Y_CHROMA : CTX_LAST_Y_LUMA);
  m.cbf = cabac + (type ? CTX_CBF_CHROMA : CTX_CBF_LUMA);
  m.root_cbf = cabac[CTX_ROOT_CBF];
  return m;
}
// the same views taken as members of the struct (the strategy kernels: this form costs their warp walks no spills)
COEFF_FN RdoqModels rdoq_models(const kvz_cuda_cabac_ctx *c, const int32_t *eb, int type)
{
  RdoqModels m;
  m.eb = eb;
  m.sig = type ? c->cu_sig_model_chroma : c->cu_sig_model_luma;
  m.one = type ? c->cu_one_model_chroma : c->cu_one_model_luma;
  m.abs = type ? c->cu_abs_model_chroma : c->cu_abs_model_luma;
  m.cg = c->cu_sig_coeff_group_model + type;
  m.last_x = type ? c->cu_ctx_last_x_chroma : c->cu_ctx_last_x_luma;
  m.last_y = type ? c->cu_ctx_last_y_chroma : c->cu_ctx_last_y_luma;
  m.cbf = type ? c->qt_cbf_model_chroma : c->qt_cbf_model_luma;
  m.root_cbf = c->cu_qt_root_cbf_model;
  return m;
}
// cost in 1/32768 bits of coding `bin` with the context whose state byte is `st` (bit 0 = MPS value)
COEFF_FN int ebits(const RdoqModels &m, int st, int bin) { return m.eb[st ^ bin]; }

// rate of the level bins of |level| given the greater1 / greater2 contexts and the Rice parameter (rdo.c:346-393)
COEFF_FN int rdoq_level_rate(const RdoqModels &m, uint32_t abs_level, int ctx_one, int ctx_abs, int rice, uint32_t c1_idx, uint32_t c2_idx)
{
  int rate = RDOQ_ONE_BIT;                                               // the sign bin
  const uint32_t base_level = (c1_idx < 8) ? (2 + (c2_idx < 1)) : 1;
  if (abs_level >= base_level) {
    int symbol = (int)(abs_level - base_level);
    if (symbol < (3 << rice)) {
      rate += ((symbol >> rice) + 1 + rice) * RDOQ_ONE_BIT;
    } else {
      int length = rice;
      symbol -= 3 << rice;
      while (symbol >= (1 << length)) symbol -= 1 << (length++);
      rate += (3 + length + 1 - rice + length) * RDOQ_ONE_BIT;
    }
    if (c1_idx < 8) {
      rate += ebits(m, m.one[ctx_one], 1);
      if (c2_idx < 1) rate += ebits(m, m.abs[ctx_abs], 1);
    }
  } else if (abs_level == 1) {
    rate += ebits(m, m.one[ctx_one], 0);
  } else if (abs_level == 2) {
    rate += ebits(m, m.one[ctx_one], 1);
    rate += ebits(m, m.abs[ctx_abs], 0);
  }
  return rate;
}

// context increment of sig_coeff_flag (context.c:366-397); map4[i] = COEFF_SIG_CTX4, wherever the caller keeps it
// (SigCtx4: a local array, which the strategy kernels' RDOQ keeps in registers)
struct SigCtx4 { COEFF_MFN int operator[](int i) const { const int map[16] = { COEFF_SIG_CTX4 }; return map[i]; } };
template <class Map4>
COEFF_FN int sig_ctx_inc(const Map4 &map4, int pattern, int scan_idx, int px, int py, int log2n, int type)
{
  if (px + py == 0) return 0;
  if (log2n == 2) return map4[4 * py + px];
  const int offset = (log2n == 3) ? (scan_idx == 0 ? 9 : 15) : (type == 0 ? 21 : 12);
  const int sx = px & 3, sy = py & 3;
  int cnt;
  if (pattern == 0) cnt = (sx + sy <= 2) ? ((sx + sy == 0) ? 2 : 1) : 0;
  else if (pattern == 1) cnt = (sy <= 1) ? ((sy == 0) ? 2 : 1) : 0;
  else if (pattern == 2) cnt = (sx <= 1) ? ((sx == 0) ? 2 : 1) : 0;
  else cnt = 2;
  return ((type == 0 && ((px >> 2) + (py >> 2)) > 0) ? 3 : 0) + offset + cnt;
}

// kvz_rdoq_sign_hiding (rdo.c:518-653) on RDOQ's output; serial, one thread.  inc / dec / sig_inc / qdelta: the
// per-position rates of kvz_sh_rates_t (rdo.h:49-58), by raster position; blk: scan position -> raster position.
template <class BlkT>
COEFF_FN void rdoq_sign_hiding(const int32_t *s_inc, const int32_t *s_dec, const int32_t *s_sig_inc, const int32_t *s_qdelta, const BlkT *blk,
                               double lambda, int bitdepth, int qp_scaled, int last_pos, const int16_t *coef, int16_t *q)
{
  const int inv_quant = inv_quant_scale(qp_scaled % 6);
  const long long rd_factor = (long long)(inv_quant * inv_quant * (1 << (2 * (qp_scaled / 6))) / lambda / 16 / (1 << (2 * (bitdepth - 8))) + 0.5);
  const int last_cg = (last_pos - 1) >> 4;
  for (int cg = last_cg; cg >= 0; --cg) {
    const BlkT *pos = blk + (cg << 4);
    int last_nz = -1, first_nz = 16;
    for (int k = 15; k >= 0; --k) if (q[pos[k]]) { last_nz = k; break; }
    for (int k = 0; k <= last_nz; ++k) if (q[pos[k]]) { first_nz = k; break; }
    if (last_nz - first_nz < 4) continue;
    const int signbit = q[pos[first_nz]] <= 0;
    unsigned sum = 0;
    for (int k = first_nz; k <= last_nz; ++k) sum += (unsigned)(int)q[pos[k]];
    if (signbit == (int)(sum & 1)) continue;
    long long best_cost = 0x7FFFFFFFFFFFFFFFLL;
    int best_pos = 0, best_change = 0;
    const int start = (cg == last_cg) ? last_nz : 15;
    for (int k = start; k >= 0; --k) {
      const int p = pos[k];
      const long long quant_cost = rd_factor * s_qdelta[p];
      const int a = iabs((int)q[p]);
      long long cost;
      int change;
      if (a != 0) {
        long long inc_bits = s_inc[p], dec_bits = s_dec[p];
        if (a == 1) dec_bits -= RDOQ_ONE_BIT + s_sig_inc[p];
        if (cg == last_cg && last_nz == k && a == 1) dec_bits -= 4 * RDOQ_ONE_BIT;
        inc_bits = -quant_cost + inc_bits;                 // PRECISION_INC = 15 - CTX_FRAC_BITS = 0
        dec_bits = quant_cost + dec_bits;
        if (inc_bits < dec_bits) { change = 1; cost = inc_bits; }
        else {
          change = -1; cost = dec_bits;
          if (k == first_nz && a == 1) cost = 0x7FFFFFFFFFFFFFFFLL;
        }
      } else {
        const int bits = RDOQ_ONE_BIT + s_inc[p] + s_sig_inc[p];
        const long long aq = quant_cost < 0 ? -quant_cost : quant_cost;
        cost = -aq + (long long)bits;
        change = 1;
        if (k < first_nz && ((coef[p] >= 0) ? 0 : 1) != signbit) cost = 0x7FFFFFFFFFFFFFFFLL;
      }
      if (cost < best_cost) { best_cost = cost; best_pos = p; best_change = change; }
    }
    if (q[best_pos] == 32767 || q[best_pos] == -32768) best_change = -1;
    if (coef[best_pos] >= 0) q[best_pos] = (int16_t)(q[best_pos] + best_change);
    else q[best_pos] = (int16_t)(q[best_pos] - best_change);
  }
}

// kvz_quant's sign-bit hiding of coefficient group g (quant-generic.c:84-176).  pos[k]: raster position of scan position
// 16 * g + k, wherever the caller takes the scan from; delta_u: the rounding remainders of kvz_quant by raster
// position; cg_nz[h]: whether group h had a non-zero level before any hiding.  Groups only interact through "is this
// the last non-zero group of the scan", so one thread per group is race free.
template <class PosT, class NzT>
COEFF_FN void quant_sign_hiding(const PosT *pos, const int16_t *coef, int16_t *q, const int32_t *delta_u, const NzT *cg_nz, int num_cg, int g)
{
  bool last_cg = true;
  for (int h = g + 1; h < num_cg; ++h) if (cg_nz[h]) { last_cg = false; break; }
  int first_nz = 16, last_nz = -1, abssum = 0;
  for (int k = 15; k >= 0; --k) if (q[pos[k]]) { last_nz = k; break; }
  for (int k = 0; k < 16; ++k) if (q[pos[k]]) { first_nz = k; break; }
  for (int k = first_nz; k <= last_nz; ++k) abssum += q[pos[k]];
  if (last_nz - first_nz < 4) return;
  const int signbit = q[pos[first_nz]] > 0 ? 0 : 1;
  if (signbit == (abssum & 1)) return;
  int min_cost = 0x7fffffff, cur_cost = 0x7fffffff, min_pos = -1;
  int final_change = 0, cur_change = 0;
  for (int k = (last_cg ? last_nz : 15); k >= 0; --k) {
    const int b = pos[k];
    if (q[b] != 0) {
      if (delta_u[b] > 0) { cur_cost = -delta_u[b]; cur_change = 1; }
      else if (k == first_nz && iabs((int)q[b]) == 1) { cur_cost = 0x7fffffff; }
      else { cur_cost = delta_u[b]; cur_change = -1; }
    } else if (k < first_nz && ((coef[b] >= 0) ? 0 : 1) != signbit) {
      cur_cost = 0x7fffffff;
    } else { cur_cost = -delta_u[b]; cur_change = 1; }
    if (cur_cost < min_cost) { min_cost = cur_cost; final_change = cur_change; min_pos = b; }
  }
  if (q[min_pos] == 32767 || q[min_pos] == -32768) final_change = -1;
  if (coef[min_pos] >= 0) q[min_pos] = (int16_t)(q[min_pos] + final_change);
  else q[min_pos] = (int16_t)(q[min_pos] - final_change);
}

// ---------------------------------------------------------------------------------------------- coefficient bits
// bits of coeff_abs_level_remaining (cabac.c:275-301)
COEFF_FN int coeff_remain_bits(int symbol, int rice)
{
  if (symbol < (3 << rice)) return (symbol >> rice) + 1 + rice;
  int length = rice;
  symbol -= 3 << rice;
  while (symbol >= (1 << length)) { symbol -= 1 << length; ++length; }
  return 3 + length + 1 - rice + length;
}

// Counting mode of the reference's coder (kvz_get_coeff_cost's CABAC branch, rdo.c:223-264: kvz_encode_coeff_nxn in
// only_count mode, encode_coding_tree-generic.c:40-290) adds kvz_f_entropy_bits[state ^ bin] = kvz_entropy_bits / 2^15
// per context-coded bin and 1 per bypass bin.  Every term is an integer multiple of 2^-15 bit, so the reference's
// double sums are exact: the walks below add integers in units of 2^-15 bit, and the caller converts the total once.
//
// A policy P says where the walk's tables and scratch live and where its bins go:
//   p.scan(scan_idx, log2n)[sp]      raster position of scan position sp
//   p.scan_cg(scan_idx, log2n)[i]    coefficient group (raster) of scan group i
//   p.group_idx(x)                   last_group(x)
//   p.sig_ctx4()                     COEFF_SIG_CTX4
//   p.abs_scratch()                  16 ints for the magnitudes of the group being counted
//   p.bin(off, val, &bits)           CABAC_FBITS_UPDATE: add the bits of `val` with model `off`, adapt when updating
//   p.trskip_enable(), p.signhide()  the configuration switches the count depends on

// the last significant position (encode_coding_tree.c:63-115) in an n x n unit, n = 1 << log2n; (lx, ly) already
// swapped for the vertical scan
template <class P>
COEFF_FN long long last_pos_bits(P &p, int lx, int ly, int n, int log2n, int type)
{
  long long bits_last = 0;
  const int idx = log2n - 2;
  const int ctx_offset = type ? 0 : (idx * 3 + (idx + 1) / 4);
  const int shift = type ? idx : (idx + 3) / 4;
  const int base_x = type ? CTX_LAST_X_CHROMA : CTX_LAST_X_LUMA;
  const int base_y = type ? CTX_LAST_Y_CHROMA : CTX_LAST_Y_LUMA;
  const int gx = p.group_idx(lx), gy = p.group_idx(ly), gmax = p.group_idx(n - 1);
  for (int k = 0; k < gx; ++k) p.bin(base_x + ctx_offset + (k >> shift), 1, &bits_last);
  if (gx < gmax) p.bin(base_x + ctx_offset + (gx >> shift), 0, &bits_last);
  for (int k = 0; k < gy; ++k) p.bin(base_y + ctx_offset + (k >> shift), 1, &bits_last);
  if (gy < gmax) p.bin(base_y + ctx_offset + (gy >> shift), 0, &bits_last);
  if (gx > 3) bits_last += (long long)((gx - 2) / 2) << 15;
  if (gy > 3) bits_last += (long long)((gy - 2) / 2) << 15;
  return bits_last;
}

// `known_cg_mask`: the raster mask of coefficient groups with a non-zero level when the caller has it, else
// COEFF_NO_MASK and the walk finds them (no unit has all 64 groups... a full 32x32 unit does: then the scan is harmless)
#define COEFF_NO_MASK 0xFFFFFFFFFFFFFFFFull
template <class P>
COEFF_FN long long coeff_bits(P &p, const int16_t *coeff, int log2n, int type, int scan_idx, int tr_skip, uint64_t known_cg_mask)
{
  const int n = 1 << log2n, side = n >> 2, ncg = side * side;
  uint64_t cg_flags = 0;                                                // sig_coeffgroup_flag, bit = cg_y * side + cg_x
  if (known_cg_mask != COEFF_NO_MASK) cg_flags = known_cg_mask;
  else for (int g = 0; g < ncg; ++g) {
    const int gy = g / side, gx = g - gy * side;
    bool any = false;
    for (int r = 0; r < 4 && !any; ++r) {
      const int16_t *row = coeff + (gy * 4 + r) * n + gx * 4;
      any = (row[0] | row[1] | row[2] | row[3]) != 0;
    }
    if (any) cg_flags |= 1ull << g;
  }
  if (!cg_flags) return 0;                                              // get_coeff_cabac_cost: no coefficients -> 0 (rdo.c:231-238)
  const auto scan = p.scan(scan_idx, log2n);
  const auto scan_cg = p.scan_cg(scan_idx, log2n);
  int cg_last = ncg - 1;
  while (!((cg_flags >> scan_cg[cg_last]) & 1)) --cg_last;
  int scan_last = cg_last * 16 + 15;
  while (!coeff[scan[scan_last]]) --scan_last;
  const int pos_last = scan[scan_last];

  long long bits = 0;                                                   // encode_coeff_nxn's accumulator
  if (n == 4 && p.trskip_enable()) p.bin(type == 0 ? CTX_TRSKIP_LUMA : CTX_TRSKIP_CHROMA, tr_skip, &bits);
  long long bits_last;                                                  // the last position has its own
  {
    int lx = pos_last & (n - 1), ly = pos_last >> log2n;
    if (scan_idx == 2) { const int t = lx; lx = ly; ly = t; }
    bits_last = last_pos_bits(p, lx, ly, n, log2n, type);
  }
  const int base_cg = CTX_SIG_CG + type;
  const int base_sig = type == 0 ? CTX_SIG_LUMA : CTX_SIG_CHROMA;
  int c1 = 1;
  int scan_pos_sig = scan_last;
  for (int i = cg_last; i >= 0; --i) {
    const int sub_pos = i << 4;
    int32_t *abs_coeff = p.abs_scratch();
    const int cg_blk = scan_cg[i];
    const int cgy = cg_blk / side, cgx = cg_blk - cgy * side;
    int last_nz = -1, first_nz = 16, num_nz = 0, rice = 0;
    if (scan_pos_sig == scan_last) {
      abs_coeff[0] = iabs((int)coeff[pos_last]);
      num_nz = 1; last_nz = scan_pos_sig; first_nz = scan_pos_sig;
      --scan_pos_sig;
    }
    const int right = (cgx < side - 1) ? (int)((cg_flags >> (cgy * side + cgx + 1)) & 1) : 0;
    const int lower = (cgy < side - 1) ? (int)((cg_flags >> ((cgy + 1) * side + cgx)) & 1) : 0;
    if (i == cg_last || i == 0) cg_flags |= 1ull << cg_blk;
    else p.bin(base_cg + (right || lower), (int)((cg_flags >> cg_blk) & 1), &bits);
    if ((cg_flags >> cg_blk) & 1) {
      const int pattern = (n == 4) ? -1 : right + (lower << 1);
      for (; scan_pos_sig >= sub_pos; --scan_pos_sig) {
        const int blk = scan[scan_pos_sig];
        const int sig = coeff[blk] != 0;
        if (scan_pos_sig > sub_pos || i == 0 || num_nz)
          p.bin(base_sig + sig_ctx_inc(p.sig_ctx4(), pattern, scan_idx, blk & (n - 1), blk >> log2n, log2n, type), sig, &bits);
        if (sig) {
          abs_coeff[num_nz++] = iabs((int)coeff[blk]);
          if (last_nz == -1) last_nz = scan_pos_sig;
          first_nz = scan_pos_sig;
        }
      }
    } else {
      scan_pos_sig = sub_pos - 1;
    }
    if (num_nz > 0) {
      const bool sign_hidden = last_nz - first_nz >= 4;
      int ctx_set = (i > 0 && type == 0) ? 2 : 0;
      if (c1 == 0) ++ctx_set;
      c1 = 1;
      const int base_one = (type == 0 ? CTX_ONE_LUMA : CTX_ONE_CHROMA) + 4 * ctx_set;
      const int num_c1 = imin(num_nz, 8);
      int first_c2 = -1;
      for (int k = 0; k < num_c1; ++k) {
        const int symbol = abs_coeff[k] > 1;
        p.bin(base_one + c1, symbol, &bits);
        if (symbol) { c1 = 0; if (first_c2 == -1) first_c2 = k; }
        else if (c1 < 3 && c1 > 0) ++c1;
      }
      if (c1 == 0 && first_c2 != -1)
        p.bin((type == 0 ? CTX_ABS_LUMA : CTX_ABS_CHROMA) + ctx_set, abs_coeff[first_c2] > 2, &bits);
      bits += (long long)((p.signhide() && sign_hidden) ? num_nz - 1 : num_nz) << 15;    // sign bins (bypass)
      if (c1 == 0 || num_nz > 8) {
        int first_coeff2 = 1;
        for (int k = 0; k < num_nz; ++k) {
          const int base_level = (k < 8) ? (2 + first_coeff2) : 1;
          if (abs_coeff[k] >= base_level) {
            bits += (long long)coeff_remain_bits(abs_coeff[k] - base_level, rice) << 15;
            if (abs_coeff[k] > 3 * (1 << rice)) rice = imin(rice + 1, 4);
          }
          if (abs_coeff[k] >= 2) first_coeff2 = 0;
        }
      }
    }
  }
  return bits_last + bits;
}

}  // namespace kvzcoeff
