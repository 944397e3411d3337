// rdoq.cuh -- rate-distortion optimised quantisation of one TU (SURVEY §8f rank 1; ref: kvz_rdoq, src/rdo.c:661-977,
// kvz_get_coded_level :395-452, kvz_get_ic_rate :346-393, calc_last_bits/get_rate_last :465-508,
// kvz_rdoq_sign_hiding :518-653, find_last_scanpos_generic quant-generic.c:376-399, context derivation
// src/context.c:315-397).
//
// The algorithm is HM's serial trellis-free RDOQ: walking the scan backwards, every coefficient picks the level
// (of at most two candidates) with the least  distortion + lambda * CABAC-rate, where the rate of a level depends on
// the greater-than-1/2 context set and Rice parameter that the previously decided levels of the coefficient group
// left behind.  That chain is serial per TU; parallelism is across TUs (a warp per TU; lane 0 walks the chain,
// all lanes do the position-parallel parts).  Costs are doubles evaluated in the reference's operation order; the
// library is built with -fmad=false, and the reference's rdo.c is plain x86-64 code without FMA contraction.
#pragma once
#include "common.cuh"
#include "transform.cuh"

namespace kvzc {

static __device__ const int32_t c_ebits_mps[64] = { COEFF_EBITS_MPS }, c_ebits_lps[64] = { COEFF_EBITS_LPS };

// The 128-entry table in the reference's indexing (state byte ^ bin), staged in shared memory by the kernels: lanes
// look up different states at the same time, which constant memory would serialise.
__device__ __forceinline__ void rdoq_load_ebits(int32_t *table /* [128] */)
{
  for (int i = threadIdx.x; i < 128; i += blockDim.x) table[i] = (i & 1) ? c_ebits_lps[i >> 1] : c_ebits_mps[i >> 1];
}

// scan position -> raster position of the 32x32 diagonal scan, shared by every 32x32 TU (filled once per process by
// rdoq_init_tables); smaller blocks build their table in shared memory
static __device__ uint16_t g_scan_diag32[1024];
static __global__ void rdoq_init_scan32_kernel() { g_scan_diag32[threadIdx.x] = (uint16_t)scan_pos(0, 5, threadIdx.x); }

// SH = sign hiding enabled: only then the per-position rate tables of kvz_sh_rates_t exist.
// cost_sig (rdo.c:683) is kept as one byte per position: the significance context (6 bits) and which of its two bin
// costs the position carries (0: flag = 0, 1: flag = 1, 2: none -- the last coefficient or a zeroed group); the double
// is lambda * entropy_bits again when the last-position search needs it.  That halves the table and lets all 32x32 TUs
// of a 1080p frame be resident at once.
template <int NN, bool SH>
struct RdoqScratch {
  double cost_coeff[NN];                                   // (the level-0 distortion cost_coeff0 is recomputed where needed)
  uint8_t sig_code[NN];
  int32_t inc[SH ? NN : 1], dec[SH ? NN : 1], sig_inc[SH ? NN : 1], qdelta[SH ? NN : 1];       // kvz_sh_rates_t (rdo.h:49-58)
  uint16_t blk[NN >= 1024 ? 1 : NN];                       // scan position -> raster position (32x32: g_scan_diag32)
  double cg_sig_cost[NN / 16];
  int32_t cg_flag[NN / 16];
  uint16_t cg_nz[NN / 16];                                 // per group: positions (bit k) whose level is non-zero
  int32_t last_x_bits[12], last_y_bits[12];
  // per coefficient group, filled by lanes 0..15 before lane 0 walks the group
  double prep_c0[16], prep_sig0[16], prep_sig1[16];
  int32_t prep_ld[16], prep_ctx_sig[16];
  int32_t best_last_p1;
};

// kvz_rdoq for one TU by one warp (all 32 lanes must call; `lane` = lane id).  coef / q: n x n row-major in shared
// memory.  type: 0 luma, 2 chroma (the reference passes 2 for U and V, quant-generic.c:239).  block_type: 1 intra,
// 2 inter.  tr_depth: depth below the CU (+1 for NxN).
//
// Work split: everything that does not depend on the serial context state is done by the lanes in parallel -- the scan
// table, the last significant position, and per coefficient group (once its neighbour pattern is known) the
// distortion of level 0 and the significance costs of its 16 positions.  Lane 0 then walks the group: level choice,
// context-set / Rice state, and the cost sums in the reference's order (double additions are not associative).
template <int NN, bool SH>
__device__ void rdoq_tu(const kvz_cuda_rdoq_params &p, const kvz_cuda_cabac_ctx *cabac, const int32_t *ebits_table, const int16_t *coef, int16_t *q, int log2n, int type,
                        int scan_idx, int block_type, int tr_depth, RdoqScratch<NN, SH> &s, int lane)
{
  const int n = 1 << log2n, nn = n * n;
  const int transform_shift = 15 - p.bitdepth - log2n;
  const int qp_scaled = scaled_qp(type, p.qp, (p.bitdepth - 8) * 6);
  const int q_bits = 14 + qp_scaled / 6 + transform_shift;
  const int qc = c_quant_scales[qp_scaled % 6];                          // flat scaling list
  const int half = 1 << (q_bits - 1);
  const double lambda = p.lambda;
  // error scale (scalinglist.c:351-368): 2^15 * 2^(-2 * transform_shift) / q / q / 2^(2 * (bitdepth - 8))
  const double err_scale = ldexp(32768.0, -2 * transform_shift) / qc / qc / (1 << (2 * (p.bitdepth - 8)));
  const RdoqModels m = rdoq_models(cabac, ebits_table, type);
  // distortion of quantising the coefficient at raster position blk to 0 (cost_coeff0, rdo.c:770-771)
  // cost_sig of a position from its code byte
  auto sig_cost_of = [&](uint8_t code) { return (code >> 6) == 2 ? 0.0 : lambda * ebits(m, m.sig[code & 63], code >> 6); };
  auto level0_cost = [&](int blk) { const double e = (double)min(abs((int)coef[blk]) * qc, 0x7FFFFFFF - half); return e * e * err_scale; };

  // ---- scan table and last significant scan position (find_last_scanpos)
  constexpr bool GLOBAL_SCAN = NN >= 1024;
  const uint16_t *blk_of = GLOBAL_SCAN ? g_scan_diag32 : s.blk;
  int my_last = -1;
  for (int sp = lane; sp < nn; sp += 32) {
    int blk;
    if constexpr (GLOBAL_SCAN) blk = blk_of[sp];
    else { blk = scan_pos(scan_idx, log2n, sp); s.blk[sp] = (uint16_t)blk; }
    const int ld = min(abs((int)coef[blk]) * qc, 0x7FFFFFFF - half);
    if (((ld + half) >> q_bits) > 0) my_last = sp;                       // increasing sp: the last assignment is the largest
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) my_last = max(my_last, __shfl_xor_sync(0xffffffffu, my_last, o));
  const int last_scanpos = my_last;
  __syncwarp();
  for (int sp = lane; sp < nn; sp += 32) if (sp > last_scanpos) q[blk_of[sp]] = 0;
  if (last_scanpos < 0) { __syncwarp(); return; }
  for (int g = lane; g < nn / 16; g += 32) { s.cg_flag[g] = 0; s.cg_sig_cost[g] = 0; }
  if (lane == 0) {
    if (SH) s.sig_inc[blk_of[last_scanpos]] = 0;
    // last-position bin costs (calc_last_bits, rdo.c:479-508)
    const int cb = log2n - 2;
    const int off = type ? 0 : (cb * 3 + ((cb + 1) >> 2));
    const int sh = type ? cb : ((cb + 3) >> 2);
    int bx = 0, by = 0, ctx;
    const int groups = last_group(n - 1);
    for (ctx = 0; ctx < groups; ++ctx) {
      const int o = off + (ctx >> sh);
      s.last_x_bits[ctx] = bx + ebits(m, m.last_x[o], 0); bx += ebits(m, m.last_x[o], 1);
      s.last_y_bits[ctx] = by + ebits(m, m.last_y[o], 0); by += ebits(m, m.last_y[o], 1);
    }
    s.last_x_bits[ctx] = bx; s.last_y_bits[ctx] = by;
  }
  __syncwarp();

  const int cg_last = last_scanpos >> 4;
  const int cgs_side = n >> 2;
  // serial state (meaningful in lane 0 only)
  int ctx_set = (last_scanpos > 0 && type == 0) ? 2 : 0;
  int c1 = 1, c2 = 0, rice = 0;
  uint32_t c1_idx = 0, c2_idx = 0;
  double base_cost = 0, block_uncoded_cost = 0;

  for (int cg = cg_last; cg >= 0; --cg) {
    const int cg_first = blk_of[cg << 4];                                  // raster position of the group's first coefficient
    const int cgx = (cg_first & (n - 1)) >> 2, cgy = (cg_first >> log2n) >> 2;
    const int cg_blk = cgy * cgs_side + cgx;
    // neighbouring coded groups: right and below (context.c:315-351); both were decided earlier in this walk
    const int right = (cgx < cgs_side - 1) ? (s.cg_flag[cgy * cgs_side + cgx + 1] != 0) : 0;
    const int lower = (cgy < cgs_side - 1) ? (s.cg_flag[(cgy + 1) * cgs_side + cgx] != 0) : 0;
    const int pattern = (n == 4) ? -1 : right + (lower << 1);
    // position-parallel part of the group: distortion of level 0, significance costs; positions that can only be
    // zero (max_abs_level == 0, rdo.c:428-432) are finished here except for their place in the ordered cost sums
    bool valid = false, cand = false;
    if (lane < 16) {
      const int sp = (cg << 4) + lane;
      if (sp <= last_scanpos) {
        valid = true;
        const int blk = blk_of[sp];
        const int ld = min(abs((int)coef[blk]) * qc, 0x7FFFFFFF - half);
        const double err = (double)ld;
        const double c0 = err * err * err_scale;
        s.prep_ld[lane] = ld;
        s.prep_c0[lane] = c0;
        cand = sp == last_scanpos || ((ld + half) >> q_bits) != 0;
        if (sp != last_scanpos) {
          const int ctx_sig = sig_ctx_inc(SigCtx4(), pattern, scan_idx, blk & (n - 1), blk >> log2n, log2n, type);
          const double sig0 = lambda * ebits(m, m.sig[ctx_sig], 0);
          s.prep_sig0[lane] = sig0;
          s.prep_sig1[lane] = lambda * ebits(m, m.sig[ctx_sig], 1);
          if (SH) s.sig_inc[blk] = ebits(m, m.sig[ctx_sig], 1) - ebits(m, m.sig[ctx_sig], 0);
          s.prep_ctx_sig[lane] = ctx_sig;
          if (!cand) {
            s.sig_code[sp] = (uint8_t)ctx_sig; s.cost_coeff[sp] = c0 + sig0;
            q[blk] = 0;
            if (SH) s.qdelta[blk] = ld >> (q_bits - 8);
          }
        }
      }
    }
    const unsigned valid_mask = __ballot_sync(0xffffffffu, valid), cand_mask = __ballot_sync(0xffffffffu, cand);
    __syncwarp();

    if (lane == 0) {
      double st_coded = 0, st_uncoded = 0, st_sig = 0, st_sig0 = 0;
      int nnz_before_pos0 = 0;
      unsigned nz_mask = 0;
      // the group's 32 inputs of the ordered sums come into registers first (independent loads), so that the walk
      // below is bound by the three addition chains only
      // (large TUs only: small ones rarely reach past their first groups, and the unrolled walk costs registers)
      constexpr bool BIG = NN >= 1024;
      double c0r[BIG ? 16 : 1], s0r[BIG ? 16 : 1];
      if constexpr (BIG) {
#pragma unroll
        for (int k = 0; k < 16; ++k) { c0r[k] = s.prep_c0[k]; s0r[k] = s.prep_sig0[k]; }
      }
#pragma unroll (BIG ? 16 : 1)
      for (int k = 15; k >= 0; --k) {
        if (!((valid_mask >> k) & 1)) continue;
        const int sp = (cg << 4) + k;
        double c0, sig0k;
        if constexpr (BIG) { c0 = c0r[k]; sig0k = s0r[k]; } else { c0 = s.prep_c0[k]; sig0k = s.prep_sig0[k]; }
        block_uncoded_cost += c0;
        if (!((cand_mask >> k) & 1)) {
          // level 0 is the only candidate: coded cost = c0 + cost of a zero significance flag
          const double cs = sig0k;
          base_cost += c0 + cs;
          st_sig += cs;
          if (k == 0) st_sig0 = cs;
          if (SH) s.inc[blk_of[sp]] = ebits(m, m.one[4 * ctx_set + c1], 0);
          if (k == 0 && sp > 0) {
            c2 = 0; rice = 0; c1_idx = 0; c2_idx = 0;
            ctx_set = (sp == 16 || type != 0) ? 0 : 2;
            if (c1 == 0) ++ctx_set;
            c1 = 1;
          }
          continue;
        }
        const int blk = blk_of[sp];
        const int ld = s.prep_ld[k];
        const uint32_t max_abs = (uint32_t)((ld + half) >> q_bits);
        const int one_ctx = 4 * ctx_set + c1, abs_ctx = ctx_set + c2;
        const bool last = sp == last_scanpos;
        // kvz_get_coded_level (rdo.c:413-452)
        uint32_t level = 0;
        double cc, cs = 0;
        int cs_kind = 2;
        if (!last && max_abs < 3) { cs = sig0k; cc = c0 + cs; cs_kind = 0; }
        else cc = 1.7e+308;
        if (max_abs != 0) {
          const double sig_now = last ? 0.0 : s.prep_sig1[k];
          const int lo = max_abs > 1 ? (int)max_abs - 1 : 1;
          for (int lvl = (int)max_abs; lvl >= lo; --lvl) {
            const double err = (double)(ld - lvl * (1 << q_bits));
            double c = err * err * err_scale + lambda * rdoq_level_rate(m, (uint32_t)lvl, one_ctx, abs_ctx, rice, c1_idx, c2_idx);
            c += sig_now;
            if (c < cc) { level = (uint32_t)lvl; cc = c; cs = sig_now; cs_kind = last ? 2 : 1; }
          }
        }
        s.cost_coeff[sp] = cc;
        s.sig_code[sp] = (uint8_t)((last ? 0 : s.prep_ctx_sig[k]) | (cs_kind << 6));
        if (SH) {
          s.qdelta[blk] = (ld - (int)level * (1 << q_bits)) >> (q_bits - 8);
          if (level > 0) {
            const int now = rdoq_level_rate(m, level, one_ctx, abs_ctx, rice, c1_idx, c2_idx);
            s.inc[blk] = rdoq_level_rate(m, level + 1, one_ctx, abs_ctx, rice, c1_idx, c2_idx) - now;
            s.dec[blk] = rdoq_level_rate(m, level - 1, one_ctx, abs_ctx, rice, c1_idx, c2_idx) - now;
          } else {
            s.inc[blk] = ebits(m, m.one[one_ctx], 0);
          }
        }
        q[blk] = (int16_t)level;
        base_cost += cc;

        const uint32_t base_level = (c1_idx < 8) ? (2 + (c2_idx < 1)) : 1;
        if (level >= base_level && level > (uint32_t)(3 * (1 << rice))) rice = min(rice + 1, 4);
        if (level >= 1) ++c1_idx;
        if (level > 1) { c1 = 0; c2 += (c2 < 2); ++c2_idx; }
        else if (c1 < 3 && c1 > 0 && level) ++c1;
        if (k == 0 && sp > 0) {                                            // context set for the next group down the scan
          c2 = 0; rice = 0; c1_idx = 0; c2_idx = 0;
          ctx_set = (sp == 16 || type != 0) ? 0 : 2;
          if (c1 == 0) ++ctx_set;
          c1 = 1;
        }
        st_sig += cs;
        if (k == 0) st_sig0 = cs;
        if (level) {
          nz_mask |= 1u << k;
          s.cg_flag[cg_blk] = 1;
          st_coded += cc - cs;
          st_uncoded += c0;
          if (k != 0) ++nnz_before_pos0;
        }
      }

      if (cg) {
        const int ctx_cg = right || lower;
        if (s.cg_flag[cg_blk] == 0) {
          s.cg_sig_cost[cg] = lambda * ebits(m, m.cg[ctx_cg], 0);
          base_cost += s.cg_sig_cost[cg] - st_sig;
        } else if (cg < cg_last) {
          if (nnz_before_pos0 == 0) { base_cost -= st_sig0; st_sig -= st_sig0; }
          double cost_zero_cg = base_cost;
          s.cg_sig_cost[cg] = lambda * ebits(m, m.cg[ctx_cg], 1);
          base_cost += s.cg_sig_cost[cg];
          cost_zero_cg += lambda * ebits(m, m.cg[ctx_cg], 0);
          cost_zero_cg += st_uncoded;
          cost_zero_cg -= st_coded;
          cost_zero_cg -= st_sig;
          if (cost_zero_cg < base_cost) {
            nz_mask = 0;
            s.cg_flag[cg_blk] = 0;
            base_cost = cost_zero_cg;
            s.cg_sig_cost[cg] = lambda * ebits(m, m.cg[ctx_cg], 0);
            for (int k = 15; k >= 0; --k) {
              const int sp = (cg << 4) + k, blk = blk_of[sp];
              if (q[blk]) { q[blk] = 0; s.cost_coeff[sp] = level0_cost(blk); s.sig_code[sp] = 2 << 6; }
            }
          }
        }
      } else {
        s.cg_flag[cg_blk] = 1;
      }
      s.cg_nz[cg] = (uint16_t)nz_mask;
    }
    __syncwarp();
  }

  if (lane == 0) {
    // ---- best last position (rdo.c:884-945)
    double best_cost;
    if (block_type != 1 && type == 0) {
      best_cost = block_uncoded_cost + lambda * ebits(m, m.root_cbf, 0);
      base_cost += lambda * ebits(m, m.root_cbf, 1);
    } else {
      const int ctx_cbf = type ? tr_depth : !tr_depth;
      best_cost = block_uncoded_cost + lambda * ebits(m, m.cbf[ctx_cbf], 0);
      base_cost += lambda * ebits(m, m.cbf[ctx_cbf], 1);
    }
    int best_last_p1 = 0;
    bool found_last = false;
    for (int cg = cg_last; cg >= 0 && !found_last; --cg) {
      const int cg_first = blk_of[cg << 4];
      const int cg_blk = ((cg_first >> log2n) >> 2) * cgs_side + ((cg_first & (n - 1)) >> 2);
      base_cost -= s.cg_sig_cost[cg];
      if (!s.cg_flag[cg_blk]) continue;
      const unsigned nz = s.cg_nz[cg];
      const int top = cg == cg_last ? (last_scanpos & 15) : 15;
      constexpr bool BIG = NN >= 1024;
      double csr[BIG ? 16 : 1];
      if constexpr (BIG) {
#pragma unroll
        for (int k = 0; k < 16; ++k) csr[k] = sig_cost_of(s.sig_code[(cg << 4) + k]);
      }
#pragma unroll (BIG ? 16 : 1)
      for (int k = 15; k >= 0; --k) {
        if (k > top) continue;
        const int sp = (cg << 4) + k;
        double csk;
        if constexpr (BIG) csk = csr[k]; else csk = sig_cost_of(s.sig_code[sp]);
        if (!((nz >> k) & 1)) { base_cost -= csk; continue; }
        const int blk = blk_of[sp];
        const int py = blk >> log2n, px = blk & (n - 1);
        const int gx = last_group(scan_idx == 2 ? py : px), gy = last_group(scan_idx == 2 ? px : py);
        double bits = s.last_x_bits[gx] + s.last_y_bits[gy];
        if (gx > 3) bits += RDOQ_ONE_BIT * ((gx - 2) >> 1);
        if (gy > 3) bits += RDOQ_ONE_BIT * ((gy - 2) >> 1);
        const double total = base_cost + lambda * bits - csk;
        if (total < best_cost) { best_last_p1 = sp + 1; best_cost = total; }
        if (q[blk] > 1) { found_last = true; break; }
        base_cost -= s.cost_coeff[sp];
        base_cost += level0_cost(blk);
      }
    }
    s.best_last_p1 = best_last_p1;
  }
  __syncwarp();

  // ---- signs and clean-up in parallel, then sign hiding
  const int best_last_p1 = s.best_last_p1;
  int abs_sum = 0;
  for (int sp = lane; sp <= last_scanpos; sp += 32) {
    const int blk = blk_of[sp];
    if (sp < best_last_p1) {
      const int level = q[blk];
      abs_sum += level;
      q[blk] = (int16_t)(coef[blk] < 0 ? -level : level);
    } else {
      q[blk] = 0;
    }
  }
  if constexpr (SH) {
    abs_sum = warp_sum(abs_sum);
    __syncwarp();
    if (lane == 0 && abs_sum >= 2) rdoq_sign_hiding(s.inc, s.dec, s.sig_inc, s.qdelta, blk_of, lambda, p.bitdepth, qp_scaled, best_last_p1, coef, q);
  }
  __syncwarp();
}

// ------------------------------------------------------------------------------------------------------------------
// One THREAD per TU, for 4x4 and 8x8 blocks: there are 10^4..10^5 of them per frame and most are empty, so running
// HM's chain once per lane beats one chain per warp.  Same arithmetic, same order; the cost tables live in the
// thread's local memory, the scan table and the entropy table in shared memory.
template <int NN, bool SH>
struct RdoqLocal {
  double cost_coeff[NN], cost_sig[NN];
  int32_t inc[SH ? NN : 1], dec[SH ? NN : 1], sig_inc[SH ? NN : 1], qdelta[SH ? NN : 1];
  double cg_sig_cost[NN / 16];
  int32_t cg_flag[NN / 16];
  int32_t last_x_bits[8], last_y_bits[8];
  const uint8_t *blk;                                      // scan position -> raster position (shared memory)
};

template <int NN, bool SH>
__device__ void rdoq_tu_thread(const kvz_cuda_rdoq_params &p, const kvz_cuda_cabac_ctx *cabac, const int32_t *ebits_table, const int16_t *coef,
                               int16_t *q, int log2n, int type, int scan_idx, int block_type, int tr_depth, RdoqLocal<NN, SH> &s)
{
  const int n = 1 << log2n;
  const int transform_shift = 15 - p.bitdepth - log2n;
  const int qp_scaled = scaled_qp(type, p.qp, (p.bitdepth - 8) * 6);
  const int q_bits = 14 + qp_scaled / 6 + transform_shift;
  const int qc = c_quant_scales[qp_scaled % 6];
  const int half = 1 << (q_bits - 1);
  const double lambda = p.lambda;
  const double err_scale = ldexp(32768.0, -2 * transform_shift) / qc / qc / (1 << (2 * (p.bitdepth - 8)));
  const RdoqModels m = rdoq_models(cabac, ebits_table, type);
  auto level_double = [&](int blk) { return min(abs((int)coef[blk]) * qc, 0x7FFFFFFF - half); };

  // find_last_scanpos (quant-generic.c:376-399)
  int last_scanpos = -1;
  for (int sp = NN - 1; sp >= 0; --sp) {
    const int blk = s.blk[sp];
    if (((level_double(blk) + half) >> q_bits) > 0) { last_scanpos = sp; break; }
    q[blk] = 0;
  }
  if (last_scanpos < 0) return;
  for (int g = 0; g < NN / 16; ++g) { s.cg_flag[g] = 0; s.cg_sig_cost[g] = 0; }
  if (SH) s.sig_inc[s.blk[last_scanpos]] = 0;
  {
    const int cb = log2n - 2;
    const int off = type ? 0 : (cb * 3 + ((cb + 1) >> 2));
    const int sh = type ? cb : ((cb + 3) >> 2);
    int bx = 0, by = 0, ctx;
    const int groups = last_group(n - 1);
    for (ctx = 0; ctx < groups; ++ctx) {
      const int o = off + (ctx >> sh);
      s.last_x_bits[ctx] = bx + ebits(m, m.last_x[o], 0); bx += ebits(m, m.last_x[o], 1);
      s.last_y_bits[ctx] = by + ebits(m, m.last_y[o], 0); by += ebits(m, m.last_y[o], 1);
    }
    s.last_x_bits[ctx] = bx; s.last_y_bits[ctx] = by;
  }

  const int cg_last = last_scanpos >> 4;
  const int cgs_side = n >> 2;
  int ctx_set = (last_scanpos > 0 && type == 0) ? 2 : 0;
  int c1 = 1, c2 = 0, rice = 0;
  uint32_t c1_idx = 0, c2_idx = 0;
  double base_cost = 0, block_uncoded_cost = 0;

  for (int cg = cg_last; cg >= 0; --cg) {
    const int cg_first = s.blk[cg << 4];
    const int cgx = (cg_first & (n - 1)) >> 2, cgy = (cg_first >> log2n) >> 2;
    const int cg_blk = cgy * cgs_side + cgx;
    const int right = (cgx < cgs_side - 1) ? (s.cg_flag[cgy * cgs_side + cgx + 1] != 0) : 0;
    const int lower = (cgy < cgs_side - 1) ? (s.cg_flag[(cgy + 1) * cgs_side + cgx] != 0) : 0;
    const int pattern = (n == 4) ? -1 : right + (lower << 1);
    double st_coded = 0, st_uncoded = 0, st_sig = 0, st_sig0 = 0;
    int nnz_before_pos0 = 0;
    for (int k = 15; k >= 0; --k) {
      const int sp = (cg << 4) + k;
      if (sp > last_scanpos) continue;
      const int blk = s.blk[sp];
      const int ld = level_double(blk);
      const uint32_t max_abs = (uint32_t)((ld + half) >> q_bits);
      const double err0 = (double)ld;
      const double c0 = err0 * err0 * err_scale;
      block_uncoded_cost += c0;
      const int one_ctx = 4 * ctx_set + c1, abs_ctx = ctx_set + c2;
      const bool last = sp == last_scanpos;
      int ctx_sig = 0;
      if (!last) {
        ctx_sig = sig_ctx_inc(SigCtx4(), pattern, scan_idx, blk & (n - 1), blk >> log2n, log2n, type);
        if (SH) s.sig_inc[blk] = ebits(m, m.sig[ctx_sig], 1) - ebits(m, m.sig[ctx_sig], 0);
      }
      uint32_t level = 0;
      double cc, cs = 0;
      if (!last && max_abs < 3) { cs = lambda * ebits(m, m.sig[ctx_sig], 0); cc = c0 + cs; }
      else cc = 1.7e+308;
      if (max_abs != 0) {
        const double sig_now = last ? 0.0 : lambda * ebits(m, m.sig[ctx_sig], 1);
        const int lo = max_abs > 1 ? (int)max_abs - 1 : 1;
        for (int lvl = (int)max_abs; lvl >= lo; --lvl) {
          const double err = (double)(ld - lvl * (1 << q_bits));
          double c = err * err * err_scale + lambda * rdoq_level_rate(m, (uint32_t)lvl, one_ctx, abs_ctx, rice, c1_idx, c2_idx);
          c += sig_now;
          if (c < cc) { level = (uint32_t)lvl; cc = c; cs = sig_now; }
        }
      }
      s.cost_coeff[sp] = cc;
      s.cost_sig[sp] = cs;
      if (SH) {
        s.qdelta[blk] = (ld - (int)level * (1 << q_bits)) >> (q_bits - 8);
        if (level > 0) {
          const int now = rdoq_level_rate(m, level, one_ctx, abs_ctx, rice, c1_idx, c2_idx);
          s.inc[blk] = rdoq_level_rate(m, level + 1, one_ctx, abs_ctx, rice, c1_idx, c2_idx) - now;
          s.dec[blk] = rdoq_level_rate(m, level - 1, one_ctx, abs_ctx, rice, c1_idx, c2_idx) - now;
        } else {
          s.inc[blk] = ebits(m, m.one[one_ctx], 0);
        }
      }
      q[blk] = (int16_t)level;
      base_cost += cc;
      const uint32_t base_level = (c1_idx < 8) ? (2 + (c2_idx < 1)) : 1;
      if (level >= base_level && level > (uint32_t)(3 * (1 << rice))) rice = min(rice + 1, 4);
      if (level >= 1) ++c1_idx;
      if (level > 1) { c1 = 0; c2 += (c2 < 2); ++c2_idx; }
      else if (c1 < 3 && c1 > 0 && level) ++c1;
      if (k == 0 && sp > 0) {
        c2 = 0; rice = 0; c1_idx = 0; c2_idx = 0;
        ctx_set = (sp == 16 || type != 0) ? 0 : 2;
        if (c1 == 0) ++ctx_set;
        c1 = 1;
      }
      st_sig += cs;
      if (k == 0) st_sig0 = cs;
      if (level) {
        s.cg_flag[cg_blk] = 1;
        st_coded += cc - cs;
        st_uncoded += c0;
        if (k != 0) ++nnz_before_pos0;
      }
    }
    if (cg) {
      const int ctx_cg = right || lower;
      if (s.cg_flag[cg_blk] == 0) {
        s.cg_sig_cost[cg] = lambda * ebits(m, m.cg[ctx_cg], 0);
        base_cost += s.cg_sig_cost[cg] - st_sig;
      } else if (cg < cg_last) {
        if (nnz_before_pos0 == 0) { base_cost -= st_sig0; st_sig -= st_sig0; }
        double cost_zero_cg = base_cost;
        s.cg_sig_cost[cg] = lambda * ebits(m, m.cg[ctx_cg], 1);
        base_cost += s.cg_sig_cost[cg];
        cost_zero_cg += lambda * ebits(m, m.cg[ctx_cg], 0);
        cost_zero_cg += st_uncoded;
        cost_zero_cg -= st_coded;
        cost_zero_cg -= st_sig;
        if (cost_zero_cg < base_cost) {
          s.cg_flag[cg_blk] = 0;
          base_cost = cost_zero_cg;
          s.cg_sig_cost[cg] = lambda * ebits(m, m.cg[ctx_cg], 0);
          for (int k = 15; k >= 0; --k) {
            const int sp = (cg << 4) + k, blk = s.blk[sp];
            if (q[blk]) { q[blk] = 0; const double e = (double)level_double(blk); s.cost_coeff[sp] = e * e * err_scale; s.cost_sig[sp] = 0; }
          }
        }
      }
    } else {
      s.cg_flag[cg_blk] = 1;
    }
  }

  // best last position (rdo.c:884-945)
  double best_cost;
  if (block_type != 1 && type == 0) {
    best_cost = block_uncoded_cost + lambda * ebits(m, m.root_cbf, 0);
    base_cost += lambda * ebits(m, m.root_cbf, 1);
  } else {
    const int ctx_cbf = type ? tr_depth : !tr_depth;
    best_cost = block_uncoded_cost + lambda * ebits(m, m.cbf[ctx_cbf], 0);
    base_cost += lambda * ebits(m, m.cbf[ctx_cbf], 1);
  }
  int best_last_p1 = 0;
  bool found_last = false;
  for (int cg = cg_last; cg >= 0 && !found_last; --cg) {
    const int cg_first = s.blk[cg << 4];
    const int cg_blk = ((cg_first >> log2n) >> 2) * cgs_side + ((cg_first & (n - 1)) >> 2);
    base_cost -= s.cg_sig_cost[cg];
    if (!s.cg_flag[cg_blk]) continue;
    for (int k = 15; k >= 0; --k) {
      const int sp = (cg << 4) + k;
      if (sp > last_scanpos) continue;
      const int blk = s.blk[sp];
      if (q[blk]) {
        const int py = blk >> log2n, px = blk & (n - 1);
        const int gx = last_group(scan_idx == 2 ? py : px), gy = last_group(scan_idx == 2 ? px : py);
        double bits = s.last_x_bits[gx] + s.last_y_bits[gy];
        if (gx > 3) bits += RDOQ_ONE_BIT * ((gx - 2) >> 1);
        if (gy > 3) bits += RDOQ_ONE_BIT * ((gy - 2) >> 1);
        const double total = base_cost + lambda * bits - s.cost_sig[sp];
        if (total < best_cost) { best_last_p1 = sp + 1; best_cost = total; }
        if (q[blk] > 1) { found_last = true; break; }
        base_cost -= s.cost_coeff[sp];
        const double e = (double)level_double(blk);
        base_cost += e * e * err_scale;
      } else {
        base_cost -= s.cost_sig[sp];
      }
    }
  }
  unsigned abs_sum = 0;
  for (int sp = 0; sp < best_last_p1; ++sp) {
    const int blk = s.blk[sp];
    const int level = q[blk];
    abs_sum += (unsigned)level;
    q[blk] = (int16_t)(coef[blk] < 0 ? -level : level);
  }
  for (int sp = best_last_p1; sp <= last_scanpos; ++sp) q[s.blk[sp]] = 0;
  if constexpr (SH) {
    if (abs_sum >= 2) rdoq_sign_hiding(s.inc, s.dec, s.sig_inc, s.qdelta, s.blk, lambda, p.bitdepth, qp_scaled, best_last_p1, coef, q);
  }
}

}  // namespace kvzc
