// ctu_search.h -- closed-loop intra search of one CTU (SURVEY §8f rank 2), all-intra slices.
//
// Restates, for the execution model of ctu_common.h:
//   search_cu / kvz_search_lcu                src/search.c:646-1068, 1209-1250   (explicit stack instead of recursion)
//   kvz_search_cu_intra, search_intra_rough,
//   search_intra_rdo, search_intra_trdepth,
//   kvz_search_cu_intra_chroma                src/search_intra.c:178-900
//   kvz_intra_recon_cu                        src/intra.c:561-698
//   kvz_quantize_lcu_residual, _trskip        src/transform.c:225-509
//   kvz_cu_rd_cost_luma / _chroma,
//   cu_rd_cost_tr_split_accurate,
//   calc_mode_bits                            src/search.c:253-582
//   kvz_mock_encode_coding_unit               src/encode_coding_tree.c:977-1075
// Scope: tr_depth_intra = 0, pu_depth_intra.min >= 1, rdo 0..3, no lossless, 8- or 10-bit 4:2:0.
//
// The mode decisions are the reference's: same candidate order, same double-precision cost expressions in the same
// operation order (the build uses -fmad=false), same CABAC model adaptation.  What differs is how the work is laid
// out: the rough search evaluates the SATD of all 35 modes in one data-parallel phase and then replays the reference's
// halving search on the table; the RDO candidates of search_intra_rdo and the colours of a CU are independent
// transform-unit jobs that run on teams sized to their units (for_tu_tasks) with private reconstructions, and only SSD / cbf / exact
// coefficient bits come back to the leader, which assembles the costs in the reference's order; each job keeps its
// reconstruction and levels in CtuWork, and the winner's are written back where the reference reconstructs the chosen
// mode once more; the cost walks that adapt the context models stay serial on the leader.
#pragma once
#include "ctu_leaf.h"

namespace kvzctu {

#define CTU_MAX_INT 0x7FFFFFFF
#define CTU_MAX_DOUBLE 1.7e+308

struct SearchFrame {
  int32_t x, y;
  int32_t stage, child;
  int32_t cbf, can_split, do_children;
  int32_t pad;
  double cost, split_cost;
  CabacState pre, post;
};

struct TuRes { int32_t ssd, has, tr_skip, pad; double bits; uint64_t cg_mask; };

template <typename Pix> struct CtuST {                       // per-CTA scalar state + scratch; shared memory on the device
  int32_t leader_tid;               // MUST be first: CTU_LEADER_TID reads it through the raw shared-memory symbol
  int32_t pad0[3];
  CabacState cabac0;                // state->cabac: the real coder's models when the CTU starts (constant)
  CabacState sc;                    // state->search_cabac
  CabacState tmp;                   // temp_cabac of the combined-CU path (search.c:989); after the search: ctu_track_models' models
  CtuConfig cfg;                    // the picture's configuration and this CTA's work area, set by ctu_job: the per-CTU
  CtuWorkT<Pix> *W;                 //   functions read them here (LDS) instead of through the caller's context
  SearchFrame fr[5];
  double ret_cost;
  IntraRefs<Pix> refs[3];
  int32_t satd[35], sad[35];
  double rc0[35], rc1[35], rmb[35];   // rough cost of a mode read with state->cabac / the search models, lambda_sqrt * mode bits
  int8_t modes[40];
  double costs[40];
  int32_t n_modes;
  int8_t cand_modes[CTU_RDO_CANDS]; // the RDO candidates in evaluation order: index into res[] and CtuWork::cand
  int8_t mpm[4];
  int8_t cmodes[8];                 // chroma candidates
  double ccosts[8];
  CuRec pred_cu;                    // the temporary CU of search_intra_rdo
  int32_t ssd[4][3];                // [leaf][colour]
  int32_t flag;
  int32_t best_mode;
  double best_cost;
  SmTables tb;
  LcuLevel<Pix> lv[5];                   // work tree: CU records here, planes in CtuWork::store
  TuRes res[CTU_RDO_CANDS][3];      // [RDO candidate][colour]
  TuRes res_ts[CTU_RDO_CANDS][2];   // [RDO candidate][transform, transform skip] of a 4x4 luma unit
  // the coefficients of the transform units reconstructed last (the CU whose cost is computed next), per colour
  int16_t stage_y[1024], stage_c[2][256];
  int32_t stage_key[3];             // (xl << 16) | (yl << 8) | depth of the staged unit, -1: none
  uint64_t stage_mask[3];           // its non-zero coefficient groups
#if defined(KVZ_CTU_PROF)
  long long prof[PR_N];
#endif
  alignas(16) unsigned char arena[CTU_ARENA_BYTES];
};
using CtuS = CtuST<uint8_t>;          // (8-bit alias, see CtuWork)

// What the CTU job is started with (ctu_job).  The functions below it take the shared state block instead and re-derive
// it with sm(): a context passed by reference would live on the caller's stack, and its pointers would be generic.
template <typename Pix> struct CtxT {
  const CtuTables *T;
  const CtuConfig *cfg;
  CtuWorkT<Pix> *W;
  CtuST<Pix> *S;
};
using Ctx = CtxT<uint8_t>;

// ------------------------------------------------------------------------------------------------ MPM, mode bits
// kvz_intra_get_dir_luma_predictor (ref: intra.c:84-127)
CTU_FN void intra_mpm(int y, const CuRec *left, const CuRec *above, int8_t *preds)
{
  int l = 1, a = 1;
  if (left && left->type == CU_INTRA) l = left->mode;
  if (above && above->type == CU_INTRA && (y & 63) != 0) a = above->mode;
  if (l == a) {
    if (l > 1) { preds[0] = (int8_t)l; preds[1] = (int8_t)(((l + 29) % 32) + 2); preds[2] = (int8_t)(((l - 1) % 32) + 2); }
    else { preds[0] = 0; preds[1] = 1; preds[2] = 26; }
  } else {
    preds[0] = (int8_t)l; preds[1] = (int8_t)a;
    if (l && a) preds[2] = 0;
    else preds[2] = (l + a) < 2 ? 26 : 1;
  }
}
// kvz_luma_mode_bits (ref: search_intra.c:641-679); leader only
template <typename Pix> CTU_FN double luma_mode_bits(CtuST<Pix> *S, int mode, const int8_t *preds)
{
  double bits = 0;
  const bool in = mode == preds[0] || mode == preds[1] || mode == preds[2];
  cabac_bin(&S->tb, &S->sc, CTX_INTRA_MODE, in, &bits);
  if (in) bits += (mode == preds[0]) ? 1 : 2;
  else bits += 5;
  return bits;
}
// kvz_chroma_mode_bits (ref: search_intra.c:682-701); leader only
template <typename Pix> CTU_FN double chroma_mode_bits(CtuST<Pix> *S, int chroma_mode, int luma_mode)
{
  double bits = 0;
  cabac_bin(&S->tb, &S->sc, CTX_CHROMA_PRED, chroma_mode != luma_mode, &bits);
  if (chroma_mode != luma_mode) bits += 2.0;
  return bits;
}

// ------------------------------------------------------------------------------------------------ work tree copies
template <typename Pix> CTU_FN void copy_cu_info(LcuLevel<Pix> *from, LcuLevel<Pix> *to, int xl, int yl, int width)
{
  const int n = width >> 2;
  #pragma unroll 1
  for (int e = CTU_TID; e < n * n; e += CTU_NT) {
    const int x = xl + 4 * (e % n), y = yl + 4 * (e / n);
    *cu_at(to, x, y) = *cu_at(from, x, y);
  }
}
template <typename Pix> CTU_FN void copy_cu_pixels(LcuLevel<Pix> *from, LcuLevel<Pix> *to, int xl, int yl, int width)
{
  #pragma unroll 1
  for (int e = CTU_TID; e < width * width; e += CTU_NT) {
    const int x = xl + e % width, y = yl + e / width;
    to->rec_y[y * 64 + x] = from->rec_y[y * 64 + x];
  }
  const int wc = width >> 1, xc = xl >> 1, yc = yl >> 1;
  #pragma unroll 1
  for (int e = CTU_TID; e < wc * wc; e += CTU_NT) {
    const int x = xc + e % wc, y = yc + e / wc;
    to->rec_u[y * 32 + x] = from->rec_u[y * 32 + x];
    to->rec_v[y * 32 + x] = from->rec_v[y * 32 + x];
  }
}
template <typename Pix> CTU_FN void copy_cu_coeffs(LcuLevel<Pix> *from, LcuLevel<Pix> *to, int xl, int yl, int width)
{
  const int zl = zorder(64, xl, yl);
  #pragma unroll 1
  for (int e = CTU_TID; e < width * width; e += CTU_NT) to->coeff_y[zl + e] = from->coeff_y[zl + e];
  const int zc = zorder(32, xl >> 1, yl >> 1), wc = width >> 1;
  #pragma unroll 1
  for (int e = CTU_TID; e < wc * wc; e += CTU_NT) { to->coeff_u[zc + e] = from->coeff_u[zc + e]; to->coeff_v[zc + e] = from->coeff_v[zc + e]; }
}
template <typename Pix> CTU_FN_NOINLINE void work_tree_copy_up(CtuST<Pix> *S, int xl, int yl, int depth)
{
  S = sm(S);
  const int w = 64 >> depth;
  PROF_T0(PR_COPY);
  copy_cu_info(&S->lv[depth + 1], &S->lv[depth], xl, yl, w);
  copy_cu_pixels(&S->lv[depth + 1], &S->lv[depth], xl, yl, w);
  copy_cu_coeffs(&S->lv[depth + 1], &S->lv[depth], xl, yl, w);
  CTU_SYNC();
  PROF_ADD(S, PR_COPY);
}
template <typename Pix> CTU_FN_NOINLINE void work_tree_copy_down(CtuST<Pix> *S, int xl, int yl, int depth)
{
  S = sm(S);
  const int w = 64 >> depth;
  PROF_T0(PR_COPY);
  for (int i = depth + 1; i <= 4; ++i) {
    copy_cu_info(&S->lv[depth], &S->lv[i], xl, yl, w);
    copy_cu_pixels(&S->lv[depth], &S->lv[i], xl, yl, w);
  }
  CTU_SYNC();
  PROF_ADD(S, PR_COPY);
}
// kvz_lcu_fill_trdepth
template <typename Pix> CTU_FN_NOINLINE void fill_trdepth(LcuLevel<Pix> *L, int xl, int yl, int depth, int tr_depth)
{
  L = sm(L);
  const int n = (64 >> depth) >> 2;
  #pragma unroll 1
  for (int e = CTU_TID; e < n * n; e += CTU_NT) cu_at(L, xl + 4 * (e % n), yl + 4 * (e / n))->tr_depth = (uint8_t)tr_depth;
  CTU_SYNC();
}
// lcu_fill_cu_info (intra fields only); `cu` may alias one of the targets
template <typename Pix> CTU_FN_NOINLINE void fill_cu_info(LcuLevel<Pix> *L, int xl, int yl, int width, const CuRec *cu)
{
  L = sm(L);
  const CuRec v = *sm(cu);
  CTU_SYNC();
  const int n = width >> 2;
  #pragma unroll 1
  for (int e = CTU_TID; e < n * n; e += CTU_NT) {
    CuRec *to = cu_at(L, xl + 4 * (e % n), yl + 4 * (e / n));
    to->type = v.type; to->depth = v.depth; to->part_size = v.part_size; to->qp = v.qp;
    to->mode = v.mode; to->mode_chroma = v.mode_chroma;
  }
  CTU_SYNC();
}

// ------------------------------------------------------------------------------------------------ transform units
CTU_FN int tu_log2(int depth, int color) { return color == 0 ? 6 - depth : (depth < 4 ? 5 - depth : 2); }
CTU_FN int stage_key_of(int xl, int yl, int depth) { return (xl << 16) | (yl << 8) | depth; }
// coefficients of the unit of `color` at (xl, yl, depth) on level L: the staged copy when it is this unit's
template <typename Pix> CTU_FN const int16_t *unit_coeffs(CtuST<Pix> *S, LcuLevel<Pix> *L, int color, int xl, int yl, int depth, uint64_t *mask)
{
  *mask = COEFF_NO_MASK;
  if (S->stage_key[color] == stage_key_of(xl, yl, depth)) { *mask = S->stage_mask[color]; return color == 0 ? S->stage_y : S->stage_c[color - 1]; }
  if (color == 0) return &L->coeff_y[zorder(64, xl, yl)];
  return (color == 1 ? L->coeff_u : L->coeff_v) + zorder(32, xl >> 1, yl >> 1);
}

template <typename Pix> CTU_FN double coeff_cost_of_unit(CtuST<Pix> *S, CabacState *sc, LcuLevel<Pix> *L, int color, int xl, int yl, int depth, int log2n, int type, int scan)
{
  uint64_t mask;
  const int16_t *co = unit_coeffs(S, L, color, xl, yl, depth, &mask);
  return coeff_cost_serial(&S->tb, &S->tb, &S->cfg, sc, co, log2n, type, scan, 0, mask);
}

// The class of a transform-unit task for for_tu_tasks: its unit's log2 side (bits 0..2) and luma or chroma.
CTU_FN int tu_class(int log2n, int color) { return log2n | (color ? 8 : 0); }

// Runs `ntasks` (at most 32) independent transform-unit jobs; class_of(t) is tu_class() of task t.  32x32 units run
// on the whole CTA, one after another.  In a batch of 4x4 units only, two consecutive tasks of the same class run on
// the two halves of one warp, so that both halves take the same path through the job (callers put such units next to
// each other: two luma units, or the U and V units of one candidate); a unit without such a neighbour leaves the other
// half idle.  Every other unit up to 16x16 runs on one warp, when four slots of the batch's largest such unit fit the
// arena (not 16x16 at 16-bit samples: then on the whole CTA as well).  The warp jobs -- a unit, or a pair of 4x4 units
// -- go to the warps in turn.  (Half-warp teams for the 4x4 and 8x8 units of mixed batches were measured slower: the
// two halves' serial sections -- RDOQ's walk, the coefficient bits -- diverge and run one after the other, so a pair
// takes about as long as two units on whole warps.)  f(team, slot base, task) must synchronise with tsync(team) only.
template <typename Pix, class K, class F> CTU_FN void for_tu_tasks(CtuST<Pix> *S, int ntasks, K class_of, F f)
{
  CTU_SYNC();
  const int nw = CTU_NWARPS;
  int lmax = 2;                     // the largest unit up to 16x16
  bool only4 = true;
  for (int t = 0; t < ntasks; ++t) {
    const int l = class_of(t) & 7;
    if (l != 2) only4 = false;
    if (l <= 4) lmax = imax(lmax, l);
  }
  const bool halves = nw > 1 && only4 && nw * 2 * tu_scratch_bytes<Pix>(16) <= CTU_ARENA_BYTES;
  const int warp_bytes = halves ? 2 * tu_scratch_bytes<Pix>(16) : tu_scratch_bytes<Pix>(1 << (2 * lmax));
  const bool warps = nw > 1 && nw * warp_bytes <= CTU_ARENA_BYTES;
  // the tasks of the CTA, of this thread's warp as a whole, of its half-warp (bit t: task t)
  unsigned cta = 0, whole = 0, half = 0;
  int job = 0;                      // warp job `job` runs on warp job % nw
  for (int t = 0; t < ntasks; ++t) {
    if ((class_of(t) & 7) > 4 || !warps) { cta |= 1u << t; continue; }
    const bool pair = halves && t + 1 < ntasks && class_of(t + 1) == class_of(t);
    if (job++ % nw == CTU_WARP) {
      if (!halves) whole |= 1u << t;
      else if (!(CTU_HALF & 1)) half |= 1u << t;
      else if (pair) half |= 2u << t;
    }
    if (pair) ++t;
  }
  if (cta) {
    const Team tm = team_cta();
    for (int t = 0; t < ntasks; ++t) if ((cta >> t) & 1) f(tm, S->arena, t);
    CTU_SYNC();
  }
  unsigned char *base = S->arena + (size_t)CTU_WARP * warp_bytes;
  if (whole) {
    const Team tm = team_warp();
    for (int t = 0; t < ntasks; ++t) if ((whole >> t) & 1) f(tm, base, t);
  }
  if (half) {
    const Team tm = team_half();
    unsigned char *slot = base + (size_t)(CTU_HALF & 1) * tu_scratch_bytes<Pix>(16);
    for (int t = 0; t < ntasks; ++t) if ((half >> t) & 1) f(tm, slot, t);
  }
  CTU_SYNC();
}
template <typename Pix, class K, class F> CTU_FN void for_tu_tasks(const CtxT<Pix> &c, int ntasks, K class_of, F f) { for_tu_tasks(sm(c.S), ntasks, class_of, f); }

template <typename Pix> CTU_FN TuS<Pix> tu_at(unsigned char *slot, int nn) { TuS<Pix> t; t.base = slot; t.nn = nn; t.ncg = nn >= 16 ? nn / 16 : 1; return t; }

// leaf part of kvz_intra_recon_cu + kvz_quantize_lcu_residual (ref: intra.c:676-696, transform.c:448-508): the
// colours of the leaf are independent jobs (prediction only reads neighbours outside the unit).
// refs_valid: bit per colour whose S->refs[] already hold this unit's references.
template <typename Pix> CTU_FN_NOINLINE void intra_recon_leaf(CtuST<Pix> *S, LcuLevel<Pix> *L, int x, int y, int depth, int mode_luma, int mode_chroma, CuRec *cur_cu, int leaf, int refs_valid)
{
  S = sm(S); L = sm(L); cur_cu = sm(cur_cu);
  const int xl = x & 63, yl = y & 63;
  CuRec *cur_tu = cu_at(L, xl, yl);
  const bool has_luma = mode_luma != -1;
  const bool has_chroma = mode_chroma != -1 && (x % 8 == 0) && (y % 8 == 0);
  const int first = has_luma ? 0 : 1, last = has_chroma ? 2 : 0;
  if (last < first) return;
  PROF_T0(PR_REFS);
  {
    int need = 0;
    for (int col = first; col <= last; ++col) if (!((refs_valid >> col) & 1)) need |= 1 << col;
    if (need) build_refs_multi(&S->tb, S->cfg.width, S->cfg.height, S->W, L, pack_log2w(tu_log2(depth, 0), tu_log2(depth, 1), tu_log2(depth, 2)), need, x, y, S->refs);
  }
  PROF_ADD(S, PR_REFS);
  // cur_pu of quantize_tr_residual: the RDOQ context selector reads its depths before the cbf bits change
  const int rdoq_tr_depth = (int)cur_cu->tr_depth - (int)cur_cu->depth + (cur_cu->part_size == SIZE_NxN ? 1 : 0);
  PROF_T0(PR_QRES4);
  // tasks luma, U, V: U and V share a warp when their units are 4x4
  for_tu_tasks(S, last - first + 1, [&](int t) { return tu_class(tu_log2(depth, first + t), first + t); }, [&](const Team &tm, unsigned char *slot, int t) {
    const int col = first + t;
    const int log2n = tu_log2(depth, col), n = 1 << log2n;
    const TuS<Pix> tu = tu_at<Pix>(slot, n * n);
    const Plane<Pix> P = plane_of(S->W, L, col);
    const int sh = col ? 1 : 0;
    const int off = (xl >> sh) + (yl >> sh) * P.lw;
    const int mode = col == 0 ? mode_luma : mode_chroma;
    // the scan follows the mode STORED in the CU record (quantize_tr_residual reads cur_pu->intra.mode_chroma, transform.c):
    // the chroma mode search predicts with its candidate while the record still holds the luma mode (bits 8.. of refs_valid)
    const int scan_mode = (col != 0 && (refs_valid >> 8)) ? (refs_valid >> 8) - 1 : mode;
    TuJob<Pix> j = { &S->refs[col], P.src + off, P.lw, col, log2n, mode, scan_order_intra(scan_mode, depth), rdoq_tr_depth };
    const int ts = tu_eval(tm, &S->tb, &S->tb, &S->cfg, S->cabac0.ctx, &S->sc, tu, j);
    // write back: reconstruction and coefficients of the level, staged copy for the cost functions
    Pix *rec = P.rec + off;
    int16_t *co = P.coeff + zorder(P.lw, xl >> sh, yl >> sh);
    const Pix *r = tu.rec();
    const int16_t *q = tu.q();
    int16_t *stage = col == 0 ? S->stage_y : S->stage_c[col - 1];
    #pragma unroll 1
    for (int e = tm.tid; e < n * n; e += tm.nt) {
      rec[(e >> log2n) * P.lw + (e & (n - 1))] = r[e];
      co[e] = q[e];
      stage[e] = q[e];
    }
    if (tm.tid == 0) {
      const TuFixed<Pix> *fx = tu.fx();
      S->res[0][col].ssd = fx->ssd; S->res[0][col].has = fx->has; S->res[0][col].tr_skip = ts;
      S->stage_key[col] = stage_key_of(xl, yl, depth);
      S->stage_mask[col] = (uint64_t)fx->cg_mask[0] | ((uint64_t)fx->cg_mask[1] << 32);
    }
    tsync(tm);
  });
  PROF_ADD_AS(S, PR_QRES4, pr_qres_of(tu_log2(depth, first)));
  CTU_LEADER {
    const bool ts_branch = depth == 4 && S->cfg.trskip_enable;       // 4x4 luma units only (transform.c:366)
    for (int col = first; col <= last; ++col) {
      cbf_clear(&cur_cu->cbf, depth, col);
      if (S->res[0][col].has) cbf_set(&cur_cu->cbf, depth, col);
      if (col == 0 && ts_branch) cur_cu->tr_skip = (uint8_t)S->res[0][0].tr_skip;
      S->ssd[leaf][col] = S->res[0][col].ssd;
    }
    if (cur_cu != cur_tu) for (int col = first; col <= last; ++col) cbf_copy(&cur_tu->cbf, cur_cu->cbf, col);
  }
  CTU_SYNC();
}

// kvz_intra_recon_cu (ref: intra.c:623-698).  cur_cu == NULL: the CU record of the level at (x, y).  Leaves the SSDs
// of the reconstructed colours in S->ssd[leaf][colour] (0 for the colours not touched).
template <typename Pix> CTU_FN_NOINLINE void intra_recon_cu(CtuST<Pix> *S, LcuLevel<Pix> *L, int x, int y, int depth, int mode_luma, int mode_chroma, CuRec *cur_cu, int refs_valid)
{
  S = sm(S); L = sm(L);
  const int xl = x & 63, yl = y & 63;
  cur_cu = cur_cu == NULL ? cu_at(L, xl, yl) : sm(cur_cu);
  CTU_LEADER {
    if (mode_luma >= 0) cbf_clear(&cur_cu->cbf, depth, 0);
    if (mode_chroma >= 0) { cbf_clear(&cur_cu->cbf, depth, 1); cbf_clear(&cur_cu->cbf, depth, 2); }
    for (int k = 0; k < 4; ++k) {
      if (mode_luma >= 0) S->ssd[k][0] = 0;
      if (mode_chroma >= 0) { S->ssd[k][1] = 0; S->ssd[k][2] = 0; }
    }
  }
  CTU_SYNC();
  if (depth == 0 || cur_cu->tr_depth > depth) {
    // with tr_depth_intra = 0 only a 64x64 CU splits, once, into its four 32x32 transform units
    const int offset = (64 >> depth) / 2;
    for (int k = 0; k < 4; ++k) {
      const int cx = x + (k & 1) * offset, cy = y + (k >> 1) * offset;
      CuRec *child = cu_at(L, cx & 63, cy & 63);
      CTU_LEADER {
        if (mode_luma >= 0) cbf_clear(&child->cbf, depth + 1, 0);
        if (mode_chroma >= 0) { cbf_clear(&child->cbf, depth + 1, 1); cbf_clear(&child->cbf, depth + 1, 2); }
      }
      CTU_SYNC();
      intra_recon_leaf(S, L, cx, cy, depth + 1, mode_luma, mode_chroma, child, k, refs_valid & ~0xFF);
    }
    CTU_LEADER {
      const uint16_t child_cbfs[3] = { cu_at(L, xl + offset, yl)->cbf, cu_at(L, xl, yl + offset)->cbf, cu_at(L, xl + offset, yl + offset)->cbf };
      if (mode_luma != -1 && depth <= 3) cbf_set_conditionally(&cur_cu->cbf, child_cbfs, depth, 0);
      if (mode_chroma != -1 && depth <= 3) { cbf_set_conditionally(&cur_cu->cbf, child_cbfs, depth, 1); cbf_set_conditionally(&cur_cu->cbf, child_cbfs, depth, 2); }
    }
    CTU_SYNC();
  } else {
    intra_recon_leaf(S, L, x, y, depth, mode_luma, mode_chroma, cur_cu, 0, refs_valid);
  }
}

// What intra_recon_cu(mode, with_chroma ? mode : -1, NULL, refs_valid) leaves for the leaf CU at (x, y, depth) that
// search_cu_intra has just evaluated at rdo >= 2 with `mode` among its RDO candidates, taken from that candidate's
// results instead of computed again: the candidate's transform-unit jobs had the same references, source, scan and
// models.  Except chroma at depth 4, which is reconstructed again: the candidate quantised it with the cbf context of
// tr_depth 1 (pred_cu of search_intra_rdo), the CU's reconstruction uses its record's tr_depth 4 - depth 3 + NxN = 2
// (rdo.c:919).
template <typename Pix> CTU_FN_NOINLINE void write_back_candidate(CtuST<Pix> *S, LcuLevel<Pix> *L, int x, int y, int depth, int mode, bool with_chroma)
{
  S = sm(S); L = sm(L);
  const int xl = x & 63, yl = y & 63;
  const int last = with_chroma && depth < 4 ? 2 : 0;
  PROF_T0(PR_WRITEBACK);
  int cand = 0;
  while (S->cand_modes[cand] != mode) ++cand;
  const bool ts_split = depth == 4 && S->cfg.trskip_enable;
  for (int col = 0; col <= last; ++col) {
    const int log2n = tu_log2(depth, col), n = 1 << log2n;
    const int unit = col == 0 ? (ts_split ? 2 * cand + S->res[cand][0].tr_skip : cand) : cand;
    const Pix *kr = (col == 0 ? S->W->cand.rec_y : S->W->cand.rec_c[col - 1]) + unit * n * n;
    const int16_t *kq = (col == 0 ? S->W->cand.q_y : S->W->cand.q_c[col - 1]) + unit * n * n;
    const Plane<Pix> P = plane_of(S->W, L, col);
    const int sh = col ? 1 : 0;
    Pix *rec = P.rec + (xl >> sh) + (yl >> sh) * P.lw;
    int16_t *co = P.coeff + zorder(P.lw, xl >> sh, yl >> sh);
    int16_t *stage = col == 0 ? S->stage_y : S->stage_c[col - 1];
    #pragma unroll 1
    for (int e = CTU_TID; e < n * n; e += CTU_NT) {
      rec[(e >> log2n) * P.lw + (e & (n - 1))] = kr[e];
      co[e] = kq[e];
      stage[e] = kq[e];
    }
  }
  CTU_LEADER {
    CuRec *cu = cu_at(L, xl, yl);
    for (int col = 0; col <= last; ++col) {
      const TuRes &r = S->res[cand][col];
      cbf_clear(&cu->cbf, depth, col);      // (the record holds the cbf bits of the candidate evaluated last)
      if (r.has) cbf_set(&cu->cbf, depth, col);
      if (col == 0 && ts_split) cu->tr_skip = (uint8_t)r.tr_skip;
      S->stage_key[col] = stage_key_of(xl, yl, depth);
      S->stage_mask[col] = r.cg_mask;
      S->ssd[0][col] = r.ssd;
      for (int k = 1; k < 4; ++k) S->ssd[k][col] = 0;
    }
  }
  CTU_SYNC();
  PROF_ADD(S, PR_WRITEBACK);
  if (with_chroma && depth == 4) intra_recon_cu(S, L, x, y, depth, -1, mode, NULL, 7);
}

// ------------------------------------------------------------------------------------------------ RD costs
// kvz_cu_rd_cost_luma for a leaf (tr_depth == depth), the search models not adapting (update == 0: the candidates of
// search_intra_rdo; the temporary CU is S->pred_cu).  Leader only.  ssd / coeff_bits: the unit's SSD and
// kvz_get_coeff_cost (0 when cbf is clear).
template <typename Pix> CTU_FN_NOINLINE double cu_rd_cost_luma_leaf(CtuST<Pix> *S, LcuLevel<Pix> *L, int xl, int yl, int depth, int ssd, double coeff_bits_y)
{
  S = sm(S); L = sm(L);
  const CuRec *pred_cu = &S->pred_cu;
  CabacState *sc = &S->sc;
  const int width = 64 >> depth;
  CuRec *tr_cu = cu_at(L, xl, yl);
  double coeff_bits = 0, tr_tree_bits = 0;
  const int tr_depth = (int)tr_cu->tr_depth - depth;
  const bool intra_split_flag = pred_cu->part_size == SIZE_NxN && depth == 3;
  const int max_tr_depth = 0 + (intra_split_flag ? 1 : 0);
  if (width <= 32 && width > 4 && !intra_split_flag && imin((int)tr_cu->tr_depth, depth) - (int)tr_cu->depth < max_tr_depth)
    cabac_bin(&S->tb, sc, CTX_TRANS_SUBDIV + (5 - (6 - depth)), tr_depth > 0, &tr_tree_bits);
  if (sc->update && tr_cu->tr_depth == tr_cu->depth) {
    const int off = CTX_CBF_CHROMA + (depth - (int)tr_cu->depth);
    cabac_bin(&S->tb, sc, off, cbf_is_set(tr_cu->cbf, depth, 1), &tr_tree_bits);
    cabac_bin(&S->tb, sc, off, cbf_is_set(tr_cu->cbf, depth, 2), &tr_tree_bits);
  }
  const int is_tr_split = (int)tr_cu->tr_depth - (int)tr_cu->depth;
  const int is_set = cbf_is_set(tr_cu->cbf, depth, 0);
  cabac_bin(&S->tb, sc, CTX_CBF_LUMA + (is_tr_split ? 0 : 1), is_set, &tr_tree_bits);     // pred_cu->type == CU_INTRA
  if (is_set) coeff_bits += coeff_bits_y;
  const double bits = tr_tree_bits + coeff_bits;
  return (double)ssd * 0.8 + bits * S->cfg.lambda;
}

// kvz_cu_rd_cost_chroma for a leaf, update == 0.  Leader only.
template <typename Pix> CTU_FN_NOINLINE double cu_rd_cost_chroma_leaf(CtuST<Pix> *S, LcuLevel<Pix> *L, int xl, int yl, int depth, const CuRec *pred_cu, int ssd, double coeff_bits_u, double coeff_bits_v)
{
  S = sm(S); L = sm(L); pred_cu = sm(pred_cu);
  CabacState *sc = &S->sc;
  CuRec *tr_cu = cu_at(L, xl, yl);
  double tr_tree_bits = 0, coeff_bits = 0;
  if (xl % 8 != 0 || yl % 8 != 0) return 0;
  const int u_is_set = cbf_is_set(tr_cu->cbf, depth, 1), v_is_set = cbf_is_set(tr_cu->cbf, depth, 2);
  if (depth < 4 && (!sc->update || tr_cu->tr_depth != tr_cu->depth)) {
    const int tr_depth = depth - (int)pred_cu->depth;
    const int off = CTX_CBF_CHROMA + tr_depth;
    if (tr_depth == 0 || cbf_is_set(tr_cu->cbf, depth - 1, 1)) cabac_bin(&S->tb, sc, off, u_is_set, &tr_tree_bits);
    if (tr_depth == 0 || cbf_is_set(tr_cu->cbf, depth - 1, 2)) cabac_bin(&S->tb, sc, off, v_is_set, &tr_tree_bits);
  }
  if (u_is_set) coeff_bits += coeff_bits_u;
  if (v_is_set) coeff_bits += coeff_bits_v;
  const double bits = tr_tree_bits + coeff_bits;
  return (double)ssd * 1.5 + bits * S->cfg.lambda;
}

// the same with the coefficient bits taken from the level's (or staged) coefficients; S->ssd[leaf] holds the SSDs
template <typename Pix> CTU_FN_NOINLINE double cu_rd_cost_chroma_leaf_of_level(CtuST<Pix> *S, LcuLevel<Pix> *L, int xl, int yl, int depth, const CuRec *pred_cu, int leaf)
{
  if (xl % 8 != 0 || yl % 8 != 0) return 0;
  S = sm(S); L = sm(L); pred_cu = sm(pred_cu);
  const CuRec *tr_cu = cu_at(L, xl, yl);
  const int width = depth <= 3 ? (64 >> (depth + 1)) : (64 >> depth);
  const int scan = scan_order_intra(pred_cu->mode_chroma, depth);
  double bu = 0, bv = 0;
  if (cbf_is_set(tr_cu->cbf, depth, 1)) bu = coeff_cost_of_unit(S, &S->sc, L, 1, xl, yl, depth, ilog2(width), 2, scan);
  if (cbf_is_set(tr_cu->cbf, depth, 2)) bv = coeff_cost_of_unit(S, &S->sc, L, 2, xl, yl, depth, ilog2(width), 2, scan);
  return cu_rd_cost_chroma_leaf(S, L, xl, yl, depth, pred_cu, S->ssd[leaf][1] + S->ssd[leaf][2], bu, bv);
}

// cu_rd_cost_tr_split_accurate (ref: search.c:414-543), one node.  Leader only.  `leaf`: index into S->ssd.  A node
// whose record is split further (tr_depth > depth) returns its tr_tree_bits only.
template <typename Pix> CTU_FN_NOINLINE double cost_accurate_node(CtuST<Pix> *S, LcuLevel<Pix> *L, int xl, int yl, int depth, const CuRec *pred_cu, int leaf)
{
  S = sm(S); L = sm(L); pred_cu = sm(pred_cu);
  CabacState *sc = &S->sc;
  const int width = 64 >> depth;
  CuRec *tr_cu = cu_at(L, xl, yl);
  double coeff_bits = 0, tr_tree_bits = 0;
  const int tr_depth = (int)tr_cu->tr_depth - depth;
  const int cb_flag_u = cbf_is_set(tr_cu->cbf, depth, 1), cb_flag_v = cbf_is_set(tr_cu->cbf, depth, 2);
  const bool intra_split_flag = pred_cu->part_size == SIZE_NxN && depth == 3;
  const int max_tr_depth = 0 + (intra_split_flag ? 1 : 0);
  if (width <= 32 && width > 4 && !intra_split_flag && imin((int)tr_cu->tr_depth, depth) - (int)tr_cu->depth < max_tr_depth)
    cabac_bin(&S->tb, sc, CTX_TRANS_SUBDIV + (5 - (6 - depth)), tr_depth > 0, &tr_tree_bits);
  {
    const int off = CTX_CBF_CHROMA + (depth - (int)tr_cu->depth);
    if ((int)tr_cu->depth == depth || cbf_is_set(tr_cu->cbf, depth - 1, 1)) cabac_bin(&S->tb, sc, off, cb_flag_u, &tr_tree_bits);
    if ((int)tr_cu->depth == depth || cbf_is_set(tr_cu->cbf, depth - 1, 2)) cabac_bin(&S->tb, sc, off, cb_flag_v, &tr_tree_bits);
  }
  if (tr_depth > 0) return tr_tree_bits;          // the caller sums the children and adds tr_tree_bits * lambda
  const int cb_flag_y = cbf_is_set(tr_cu->cbf, depth, 0);
  const int is_tr_split = depth - (int)tr_cu->depth;
  cabac_bin(&S->tb, sc, CTX_CBF_LUMA + (is_tr_split ? 0 : 1), cb_flag_y, &tr_tree_bits);   // CU_INTRA
  const unsigned luma_ssd = (unsigned)S->ssd[leaf][0];
  if (cb_flag_y) {
    const int scan = scan_order_intra(pred_cu->mode, depth);
    coeff_bits += coeff_cost_of_unit(S, sc, L, 0, xl, yl, depth, ilog2(width), 0, scan);
  }
  unsigned chroma_ssd = 0;
  if (xl % 8 == 0 && yl % 8 == 0) {
    const int chroma_width = depth <= 3 ? (64 >> (depth + 1)) : (64 >> depth);
    chroma_ssd = (unsigned)S->ssd[leaf][1] + (unsigned)S->ssd[leaf][2];
    const int scan = scan_order_intra(pred_cu->mode_chroma, depth);
    if (cb_flag_u) coeff_bits += coeff_cost_of_unit(S, sc, L, 1, xl, yl, depth, ilog2(chroma_width), 2, scan);
    if (cb_flag_v) coeff_bits += coeff_cost_of_unit(S, sc, L, 2, xl, yl, depth, ilog2(chroma_width), 2, scan);
  }
  const double bits = tr_tree_bits + coeff_bits;
  return luma_ssd * 0.8 + chroma_ssd * 1.5 + bits * S->cfg.lambda;
}
template <typename Pix> CTU_FN_NOINLINE double cost_tr_split_accurate(CtuST<Pix> *S, LcuLevel<Pix> *L, int xl, int yl, int depth, const CuRec *pred_cu)
{
  S = sm(S); L = sm(L);
  const bool split = (int)cu_at(L, xl, yl)->tr_depth > depth;       // (the cost walks do not change the records)
  const double v = cost_accurate_node(S, L, xl, yl, depth, pred_cu, 0);
  if (!split) return v;
  const int offset = 64 >> (depth + 1);
  double sum = 0;
  for (int k = 0; k < 4; ++k) sum += cost_accurate_node(S, L, xl + (k & 1) * offset, yl + (k >> 1) * offset, depth + 1, pred_cu, k);
  return sum + v * S->cfg.lambda;
}

// calc_mode_bits (ref: search.c:557-582).  Leader only.
template <typename Pix> CTU_FN double calc_mode_bits(CtuST<Pix> *S, LcuLevel<Pix> *L, const CuRec *cur_cu, int x, int y)
{
  const int xl = x & 63, yl = y & 63;
  int8_t cand[3];
  const CuRec *left = x >= 4 ? cu_at(L, xl - 4, yl) : NULL;
  const CuRec *above = y >= 4 ? cu_at(L, xl, yl - 4) : NULL;
  intra_mpm(y, left, above, cand);
  double mode_bits = luma_mode_bits(S, cur_cu->mode, cand);
  if (x % 8 == 0 && y % 8 == 0) mode_bits += chroma_mode_bits(S, cur_cu->mode_chroma, cur_cu->mode);
  return mode_bits;
}

// kvz_mock_encode_coding_unit for an intra CU in an I slice (ref: encode_coding_tree.c:977-1075, 464-652, 672-743).
// Leader only.
template <typename Pix> CTU_FN_NOINLINE double mock_encode_coding_unit(CtuST<Pix> *S, LcuLevel<Pix> *L, int x, int y, int depth, const CuRec *cur_cu)
{
  S = sm(S); L = sm(L); cur_cu = sm(cur_cu);
  double bits = 0;
  CabacState *sc = &S->sc;
  const int xl = x & 63, yl = y & 63;
  const int cu_width = 64 >> depth;
  const CuRec *left_cu = x ? cu_at(L, xl - 1, yl) : NULL;
  const CuRec *above_cu = y ? cu_at(L, xl, yl - 1) : NULL;
  const bool border = S->cfg.width < x + cu_width || S->cfg.height < y + cu_width;
  if (depth != 3 && !border) {
    int split_model = 0;
    if (left_cu && left_cu->depth > depth) ++split_model;
    if (above_cu && above_cu->depth > depth) ++split_model;
    cabac_bin(&S->tb, sc, CTX_SPLIT + split_model, 0, &bits);
  }
  // kvz_encode_part_mode
  {
    double pb = 0;
    if (depth == 3) cabac_bin(&S->tb, sc, CTX_PART_SIZE, cur_cu->part_size == SIZE_2Nx2N ? 1 : 0, &pb);
    bits += pb;
  }
  // encode_intra_coding_unit in counting mode
  const int num_pu = cur_cu->part_size == SIZE_NxN ? 4 : 1;
  unsigned flag = 0, mpm_nz = 0;    // bit j: PU j's mode is an MPM, it is not the first MPM
  int mode0 = 0;
  for (int j = 0; j < num_pu; ++j) {
    const int pw = num_pu == 4 ? cu_width / 2 : cu_width;
    const int pu_x = x + (num_pu == 4 ? (j & 1) * pw : 0), pu_y = y + (num_pu == 4 ? (j >> 1) * pw : 0);
    const CuRec *cur_pu = cu_at(L, pu_x & 63, pu_y & 63);
    // the reference takes SUB_SCU(pu_x - 1): at the CTU's left edge this is the CTU's own last column
    const CuRec *left_pu = pu_x > 0 ? cu_at(L, (pu_x - 1) & 63, pu_y & 63) : NULL;
    const CuRec *above_pu = ((pu_y & 63) > 0 && pu_y > 0) ? cu_at(L, pu_x & 63, (pu_y - 1) & 63) : NULL;
    int8_t preds[3];
    intra_mpm(pu_y, left_pu, above_pu, preds);
    const int mode = cur_pu->mode;
    if (j == 0) mode0 = mode;
    int mpm_idx = -1;
    for (int i = 0; i < 3; ++i) if (preds[i] == mode) { mpm_idx = i; break; }
    if (mpm_idx != -1) flag |= 1u << j;
    if (mpm_idx > 0) mpm_nz |= 1u << j;
  }
  for (int j = 0; j < num_pu; ++j) cabac_bin(&S->tb, sc, CTX_INTRA_MODE, (flag >> j) & 1, &bits);
  for (int j = 0; j < num_pu; ++j) {
    if ((flag >> j) & 1) { bits += 1; if ((mpm_nz >> j) & 1) bits += 1; }
    else bits += 5;
  }
  {
    const int mc = cur_cu->mode_chroma;
    if (mc == mode0) cabac_bin(&S->tb, sc, CTX_CHROMA_PRED, 0, &bits);
    else { cabac_bin(&S->tb, sc, CTX_CHROMA_PRED, 1, &bits); bits += 2; }
  }
  return bits;
}

// ------------------------------------------------------------------------------------------------ intra mode search
// kvz_sort_modes: insertion sort, stable for equal costs
CTU_FN void sort_modes(int8_t *modes, double *costs, int length)
{
  for (int i = 1; i < length; ++i) {
    const double cur_cost = costs[i];
    const int8_t cur_mode = modes[i];
    int j = i;
    while (j > 0 && cur_cost < costs[j - 1]) { costs[j] = costs[j - 1]; modes[j] = modes[j - 1]; --j; }
    costs[j] = cur_cost; modes[j] = cur_mode;
  }
}

// The per-mode quantities of search_intra_rough (get_cost / get_cost_dual, search_intra.c:89-160, and the mode bits
// added at :524) for all 35 modes, one mode per thread.
template <typename Pix> CTU_FN_NOINLINE void rough_mode_costs(CtuST<Pix> *S, int log2w)
{
  S = sm(S);
  const int8_t *mpm = S->mpm;
  const CtuConfig *cfg = &S->cfg;
  const bool ts = log2w == 2 && cfg->trskip_enable;
  #pragma unroll 1
  for (int mode = CTU_TID; mode < 35; mode += CTU_NT) {
    // get_cost_dual reads state->cabac, get_cost reads state->search_cabac (search_intra.c:102, 142)
    for (int k = 0; k < 2; ++k) {
      const CabacState *cb = k == 0 ? &S->cabac0 : &S->sc;
      double cost = (double)(unsigned)S->satd[mode];
      if (ts) {
        double b = (double)S->tb.ebits[cb->ctx[CTX_TRSKIP_LUMA] ^ 1] * (1.0 / 32768.0) - (double)S->tb.ebits[cb->ctx[CTX_TRSKIP_LUMA] ^ 0] * (1.0 / 32768.0);
        b += 2.0 * ((double)S->tb.ebits[cb->ctx[CTX_TRSKIP_CHROMA] ^ 1] * (1.0 / 32768.0) - (double)S->tb.ebits[cb->ctx[CTX_TRSKIP_CHROMA] ^ 0] * (1.0 / 32768.0));
        const double sad_cost = 1.7 * (double)(unsigned)S->sad[mode] + cfg->lambda_sqrt * b;
        if (sad_cost < cost) cost = sad_cost;
      }
      (k == 0 ? S->rc0 : S->rc1)[mode] = cost;
    }
    // kvz_luma_mode_bits (the models do not adapt here: update == 0)
    double bits = 0;
    const bool in = mode == mpm[0] || mode == mpm[1] || mode == mpm[2];
    bits += (double)S->tb.ebits[S->sc.ctx[CTX_INTRA_MODE] ^ (in ? 1 : 0)] * (1.0 / 32768.0);
    if (in) bits += (mode == mpm[0]) ? 1 : 2;
    else bits += 5;
    S->rmb[mode] = cfg->lambda_sqrt * bits;
  }
  CTU_SYNC();
}

// search_intra_rough (ref: search_intra.c:391-530) replayed on the per-mode tables.  Leader only.
template <typename Pix> CTU_FN_NOINLINE int rough_search_replay(CtuST<Pix> *S, int log2w)
{
  S = sm(S);
  const int8_t *mpm = S->mpm;
  const CtuConfig *cfg = &S->cfg;
  int8_t *modes = S->modes;
  double *costs = S->costs;
  int n = 0;
  uint64_t present = 0;           // modes already in the list
  int32_t min_cost = CTU_MAX_INT, max_cost = -CTU_MAX_INT - 1;
  int offset;
  if (cfg->full_intra_search) offset = 1;
  else offset = log2w == 2 ? 2 : (log2w == 3 ? 4 : 8);
  int best_mode = 2;
  double best_of_list = CTU_MAX_DOUBLE;
  for (int mode = 2; mode <= 34; mode += offset) {      // (mode, mode + offset) pairs of the reference's loop, in its order
    const double cst = S->rc0[mode];
    costs[n] = cst;
    modes[n] = (int8_t)mode;
    present |= 1ull << mode;
    // the reference keeps min / max as int32 (implicit conversion of the double cost)
    min_cost = imin(min_cost, (int32_t)cst);
    max_cost = imax(max_cost, (int32_t)cst);
    if (cst < best_of_list) { best_of_list = cst; best_mode = mode; }     // first minimum, as select_best_mode_index
    ++n;
  }
  double best_cost = min_cost;
  if (min_cost != max_cost) {
    while (offset > 1) {
      offset >>= 1;
      const int center = best_mode;
      const int test[2] = { center - offset, center + offset };
      #pragma unroll
      for (int i = 0; i < 2; ++i) {
        if (test[i] >= 2 && test[i] <= 34) {
          costs[n] = S->rc0[test[i]];
          modes[n] = (int8_t)test[i];
          present |= 1ull << test[i];
          if (costs[n] < best_cost) { best_cost = costs[n]; best_mode = modes[n]; }
          ++n;
        }
      }
    }
  }
  const int add_modes[5] = { mpm[0], mpm[1], mpm[2], 0, 1 };
  #pragma unroll
  for (int p = 0; p < 5; ++p) {
    if (!((present >> add_modes[p]) & 1)) { costs[n] = S->rc1[add_modes[p]]; modes[n] = (int8_t)add_modes[p]; present |= 1ull << add_modes[p]; ++n; }
  }
  for (int i = 0; i < n; ++i) costs[i] += S->rmb[modes[i]];
  return n;
}

// copy of a transform-unit job's reconstruction and levels (team)
template <typename Pix> CTU_FN_NOINLINE void keep_unit(Team tm, TuS<Pix> tu, Pix *kr, int16_t *kq)
{
  tu.base = sm(tu.base);
  const Pix *r = tu.rec();
  const int16_t *q = tu.q();
  #pragma unroll 1
  for (int e = tm.tid; e < tu.nn; e += tm.nt) { kr[e] = r[e]; kq[e] = q[e]; }
}

// kvz_search_cu_intra (ref: search_intra.c:806-900): best luma mode of the CU at (x, y, depth) on level L.
// Result in S->best_mode / S->best_cost.
template <typename Pix> CTU_FN_NOINLINE void search_cu_intra(CtuST<Pix> *S, LcuLevel<Pix> *L, int x, int y, int depth)
{
  S = sm(S); L = sm(L);
  const CtuConfig *cfg = &S->cfg;
  const int xl = x & 63, yl = y & 63;
  const int log2w = 6 - depth;
  CTU_LEADER {
    const CuRec *left = x >= 4 ? cu_at(L, xl - 1, yl) : NULL;
    const CuRec *above = (y >= 4 && yl > 0) ? cu_at(L, xl, yl - 1) : NULL;
    intra_mpm(y, left, above, S->mpm);
  }
  CTU_SYNC();
  PROF_T0(PR_REFS);
  {
    // luma for the rough search; the chroma references the CU's reconstruction (and RDO candidates) will need as well
    build_refs_multi(&S->tb, cfg->width, cfg->height, S->W, L, pack_log2w(log2w, tu_log2(depth, 1), tu_log2(depth, 2)), ((x & 4) || (y & 4)) ? 1 : 7, x, y, S->refs);
  }
  PROF_ADD(S, PR_REFS);
  // rough search: SATD (and SAD for 4x4 transform-skip candidates) of every mode, then the reference's selection
  PROF_T0(PR_SATD);
  rough_costs_all_modes(&S->refs[0], (RoughExt<Pix> *)S->arena, log2w, 0, &S->W->src_y[yl * 64 + xl], 64, S->satd, S->sad, log2w == 2 && cfg->trskip_enable);
  PROF_ADD(S, PR_SATD);
  PROF_T0(PR_REPLAY);
  rough_mode_costs(S, log2w);
  CTU_LEADER S->n_modes = rough_search_replay(S, log2w);
  CTU_SYNC();
  PROF_ADD(S, PR_REPLAY);
  PROF_T0(PR_RDO_LOOP);
  fill_trdepth(L, xl, yl, depth, depth);
  if (cfg->rdo >= 2) {
    // search_intra_rdo (ref: search_intra.c:558-638) with tr_depth == depth
    CTU_LEADER {
      const int to_search = depth == 4 ? 3 : 2;
      int check = imin(S->n_modes, to_search);
      sort_modes(S->modes, S->costs, S->n_modes);
      for (int p = 0; p < 3; ++p) {
        bool found = false;
        for (int r = 0; r < check; ++r) if (S->mpm[p] == S->modes[r]) { found = true; break; }
        if (!found) { S->modes[check] = S->mpm[p]; ++check; }
      }
      S->n_modes = check;
    }
    CTU_SYNC();
    const bool reconstruct_chroma = !((x & 4) || (y & 4));
    const int np = reconstruct_chroma ? 3 : 1;
    // The candidates (search_intra_trdepth's no-split branch, tr_depth == depth) are independent of each other and so
    // are their colours: every (candidate, colour) pair is one transform-unit job with a private reconstruction.  The
    // temporary CU of the reference (pred_cu: depth = tr_depth = `depth`, NxN at depth 4) only matters through RDOQ's
    // cbf context and the cbf bits collected below.
    const int ncand = S->n_modes;
    const int rdoq_tr_depth = depth == 4 ? 1 : 0;
    PROF_T0(PR_QRES4);
    // 4x4 luma units with transform skip enabled: the two alternatives of kvz_quantize_residual_trskip are jobs of their
    // own (better balance over the warps), the leader picks below; the pick's coefficient bits are the ones its luma
    // cost needs (same call: rdo.c:251-258 codes tr_skip as 0), so they are not computed a third time
    const bool ts_split = depth == 4 && cfg->trskip_enable;
    const int nluma = ts_split ? 2 : 1;
    // tasks: the luma units of all candidates (k: the transform-skip alternative), then (U, V) of each candidate, so
    // that the two halves of a warp get two luma units or the two chroma units of one candidate
    const int ntl = ncand * nluma;
    for_tu_tasks(S, ntl + ncand * (np - 1), [&](int t) { return t < ntl ? tu_class(log2w, 0) : tu_class(tu_log2(depth, 1), 1); },
                 [&](const Team &tm, unsigned char *slot, int t) {
      const int cand = t < ntl ? t / nluma : (t - ntl) >> 1;
      const int k = t < ntl ? t - cand * nluma : 0;
      const int col = t < ntl ? 0 : 1 + ((t - ntl) & 1);
      const int mode = S->modes[cand];
      const int log2n = tu_log2(depth, col), n = 1 << log2n;
      const TuS<Pix> tu = tu_at<Pix>(slot, n * n);
      const Plane<Pix> P = plane_of(S->W, L, col);
      const int sh = col ? 1 : 0;
      const int off = (xl >> sh) + (yl >> sh) * P.lw;
      TuJob<Pix> j = { &S->refs[col], P.src + off, P.lw, col, log2n, mode, scan_order_intra(mode, depth), rdoq_tr_depth };
      int ts = 0;
      if (col == 0 && ts_split) tu_core(tm, &S->tb, &S->tb, cfg, S->cabac0.ctx, tu, j, k == 1);
      else ts = tu_eval(tm, &S->tb, &S->tb, cfg, S->cabac0.ctx, &S->sc, tu, j);
      // keep the unit for write_back_candidate (not the chroma of depth 4, which is quantised again: see there)
      if (col == 0 || depth < 4) {
        const int unit = col == 0 ? cand * nluma + k : cand;
        Pix *kr = (col == 0 ? S->W->cand.rec_y : S->W->cand.rec_c[col - 1]) + unit * n * n;
        int16_t *kq = (col == 0 ? S->W->cand.q_y : S->W->cand.q_c[col - 1]) + unit * n * n;
        keep_unit(tm, tu, kr, kq);
      }
      if (tm.tid == 0) {
        const TuFixed<Pix> *fx = tu.fx();
        TuRes *r = (col == 0 && ts_split) ? &S->res_ts[cand][k] : &S->res[cand][col];
        r->ssd = fx->ssd; r->has = fx->has; r->tr_skip = ts;
        r->cg_mask = (uint64_t)fx->cg_mask[0] | ((uint64_t)fx->cg_mask[1] << 32);
        // coefficient bits of kvz_cu_rd_cost_luma / _chroma: the search models are not adapted here (update == 0)
        PROF_T0(PR_COEFFCOST);
        r->bits = fx->has ? coeff_cost_serial(&S->tb, &S->tb, cfg, &S->sc, tu.q(), log2n, col ? 2 : 0, j.scan_idx, 0, r->cg_mask) : 0.0;
        PROF_ADD(S, PR_COEFFCOST);
      }
      tsync(tm);
    });
    PROF_ADD_AS(S, PR_QRES4, pr_qres_of(log2w));
    PROF_T0(PR_COST);
    int checked = ncand;
    CTU_LEADER {
      CuRec *tr_cu = cu_at(L, xl, yl);
      tr_cu->tr_depth = (uint8_t)depth;
      for (int r = 0; r < ncand; ++r) {
        if (ts_split) {
          // kvz_quantize_residual_trskip (transform.c:242-288): SSD + coefficient bits * lambda, transform skip only if cheaper
          double tc[2];
          for (int k = 0; k < 2; ++k) { tc[k] = (double)(unsigned)S->res_ts[r][k].ssd; tc[k] += S->res_ts[r][k].bits * cfg->lambda; }
          const int pick = tc[0] <= tc[1] ? 0 : 1;
          S->res[r][0] = S->res_ts[r][pick];
          S->res[r][0].tr_skip = pick;
        }
        const int mode = S->modes[r];
        const double rdo_bitcost = luma_mode_bits(S, mode, S->mpm);
        S->costs[r] = rdo_bitcost * cfg->lambda;
        CuRec *p = &S->pred_cu;
        p->depth = (uint8_t)depth; p->type = CU_INTRA; p->part_size = depth == 4 ? SIZE_NxN : SIZE_2Nx2N;
        p->mode = (int8_t)mode; p->mode_chroma = (int8_t)mode; p->cbf = 0; p->tr_depth = (uint8_t)depth;
        for (int col = 0; col < np; ++col) if (S->res[r][col].has) cbf_set(&p->cbf, depth, col);
        // the level's record carries the candidate's cbf bits (cbf_copy in kvz_intra_recon_cu's leaf)
        for (int col = 0; col < np; ++col) cbf_copy(&tr_cu->cbf, p->cbf, col);
        double nosplit = 0.0;
        nosplit += cu_rd_cost_luma_leaf(S, L, xl, yl, depth, S->res[r][0].ssd, S->res[r][0].bits);
        if (reconstruct_chroma) nosplit += cu_rd_cost_chroma_leaf(S, L, xl, yl, depth, p, S->res[r][1].ssd + S->res[r][2].ssd, S->res[r][1].bits, S->res[r][2].bits);
        S->costs[r] += nosplit;
        if (cfg->intra_rdo_et && !cbf_is_set_any(p->cbf, depth)) { S->n_modes = r + 1; break; }
      }
    }
    CTU_SYNC();
    PROF_ADD(S, PR_COST);
    checked = S->n_modes;
    CTU_LEADER {
      for (int r = 0; r < checked; ++r) S->cand_modes[r] = S->modes[r];
      S->n_modes = checked;
      sort_modes(S->modes, S->costs, checked);
    }
    CTU_SYNC();
  }
  PROF_ADD(S, PR_RDO_LOOP);
  CTU_LEADER {
    int bi = 0;
    for (int i = 1; i < S->n_modes; ++i) if (S->costs[i] < S->costs[bi]) bi = i;
    S->best_mode = S->modes[bi];
    S->best_cost = S->costs[bi];
  }
  CTU_SYNC();
}

// kvz_search_cu_intra_chroma (ref: search_intra.c:748-803) for rdo 2..3 (num_modes = 2).  Returns the mode (uniform).
template <typename Pix> CTU_FN_NOINLINE int search_cu_intra_chroma(CtuST<Pix> *S, LcuLevel<Pix> *L, int x, int y, int depth)
{
  S = sm(S); L = sm(L);
  const int xl = x & 63, yl = y & 63;
  const int intra_mode = cu_at(L, xl, yl)->mode;
  const int log2wc = imax(6 - depth - 1, 2);
  const int wc = 1 << log2wc;
  CTU_LEADER {
    const int8_t init[5] = { 0, 26, 10, 1, 34 };
    #pragma unroll
    for (int i = 0; i < 5; ++i) S->cmodes[i] = init[i];
    if (intra_mode != 0 && intra_mode != 26 && intra_mode != 10 && intra_mode != 1) S->cmodes[4] = (int8_t)intra_mode;
  }
  CTU_SYNC();
  build_refs(&S->tb, &S->cfg, S->W, L, log2wc, 1, x, y, &S->refs[1]);
  build_refs(&S->tb, &S->cfg, S->W, L, log2wc, 2, x, y, &S->refs[2]);
  // search_intra_chroma_rough: SATD of the five candidates on U and V (the luma mode is skipped: cost 0)
  const int ci = (yl >> 1) * 32 + (xl >> 1);
  rough_costs_all_modes(&S->refs[1], (RoughExt<Pix> *)S->arena, log2wc, 1, &S->W->src_u[ci], 32, S->satd, S->sad, false);
  CTU_LEADER { for (int i = 0; i < 5; ++i) S->ccosts[i] = 0; for (int i = 0; i < 5; ++i) if (S->cmodes[i] != intra_mode) S->ccosts[i] += (double)(unsigned)S->satd[S->cmodes[i]]; }
  CTU_SYNC();
  rough_costs_all_modes(&S->refs[2], (RoughExt<Pix> *)S->arena, log2wc, 2, &S->W->src_v[ci], 32, S->satd, S->sad, false);
  CTU_LEADER {
    for (int i = 0; i < 5; ++i) if (S->cmodes[i] != intra_mode) S->ccosts[i] += (double)(unsigned)S->satd[S->cmodes[i]];
    sort_modes(S->cmodes, S->ccosts, 5);
  }
  CTU_SYNC();
  (void)wc;
  // kvz_search_intra_chroma_rdo over the two best
  double best_cost = CTU_MAX_INT;
  int best_mode = 0;
  for (int i = 0; i < 2; ++i) {
    const int mode = S->cmodes[i];
    intra_recon_cu(S, L, x, y, depth, -1, mode, NULL, (depth == 0 ? 0 : 6) | ((intra_mode + 1) << 8));
    CTU_LEADER {
      CuRec *tr_cu = cu_at(L, xl, yl);
      double cost;
      if (depth == 0) {
        // kvz_cu_rd_cost_chroma recursion over the four 32x32 quadrants (ref: search.c:377-388)
        CabacState *sc = &S->sc;
        double tr_tree_bits = 0;
        if (!sc->update || tr_cu->tr_depth != tr_cu->depth) {
          cabac_bin(&S->tb, sc, CTX_CBF_CHROMA, cbf_is_set(tr_cu->cbf, 0, 1), &tr_tree_bits);
          cabac_bin(&S->tb, sc, CTX_CBF_CHROMA, cbf_is_set(tr_cu->cbf, 0, 2), &tr_tree_bits);
        }
        double sum = 0;
        for (int k = 0; k < 4; ++k) sum += cu_rd_cost_chroma_leaf_of_level(S, L, xl + (k & 1) * 32, yl + (k >> 1) * 32, 1, tr_cu, k);
        cost = sum + tr_tree_bits * S->cfg.lambda;
      } else {
        cost = cu_rd_cost_chroma_leaf_of_level(S, L, xl, yl, depth, tr_cu, 0);
      }
      const double mode_bits = chroma_mode_bits(S, mode, intra_mode);
      cost += mode_bits * S->cfg.lambda;
      S->ccosts[5 + i] = cost;
    }
    CTU_SYNC();
    if (S->ccosts[5 + i] < best_cost) { best_cost = S->ccosts[5 + i]; best_mode = mode; }
  }
  return best_mode;
}

// ------------------------------------------------------------------------------------------------ search_cu
template <typename Pix> CTU_FN int split_model_of(LcuLevel<Pix> *L, int x, int y, int depth)     // get_ctx_cu_split_model (search.c:634-641)
{
  const int xl = x & 63, yl = y & 63;
  const bool condA = x >= 8 && cu_at(L, xl - 1, yl)->depth > depth;
  const bool condL = y >= 8 && cu_at(L, xl, yl - 1)->depth > depth;
  return (condA ? 1 : 0) + (condL ? 1 : 0);
}

// search_cu for the whole CTU at (cx, cy) (luma picture coordinates); returns with the decisions on level 0.  The
// caller has loaded the tables into S->tb.
template <typename Pix> CTU_FN_NOINLINE void search_ctu(CtuST<Pix> *S, int cx, int cy)
{
  S = sm(S);
  const CtuConfig *cfg = &S->cfg;
  CTU_LEADER { S->fr[0].x = cx; S->fr[0].y = cy; S->fr[0].stage = 0; S->stage_key[0] = S->stage_key[1] = S->stage_key[2] = -1; }
  CTU_SYNC();
  int d = 0;
  for (;;) {
    SearchFrame *F = &S->fr[d];
    LcuLevel<Pix> *L = &S->lv[d];
    // Every thread takes its copy of the frame's state, THEN the barrier: the leader changes that state below, and a
    // thread that read it late would take another branch than the others (all control flow here must be uniform).
    const int x = F->x, y = F->y;
    const int stage = F->stage;
    const bool descend = F->do_children && F->child < 4 && F->split_cost < F->cost;
    const int next_child = F->child;
    CTU_SYNC();
    const int xl = x & 63, yl = y & 63;
    const int cu_width = 64 >> d;
    if (stage == 0) {
      // ---------------- entry: this depth's own mode decision
      if (x >= cfg->width || y >= cfg->height) {
        CTU_LEADER { S->ret_cost = 0; }
        CTU_SYNC();
        if (d == 0) break;
        --d;
        CTU_LEADER { S->fr[d].split_cost += S->ret_cost; }
        CTU_SYNC();
        continue;
      }
      CuRec *cur_cu = cu_at(L, xl, yl);
      CTU_LEADER {
        F->pre = S->sc;
        F->cost = CTU_MAX_DOUBLE;
        cur_cu->depth = (uint8_t)(d > 3 ? 3 : d);
        cur_cu->tr_depth = (uint8_t)(d > 0 ? d : 1);
        cur_cu->type = CU_NOTSET;
        cur_cu->part_size = SIZE_2Nx2N;
        cur_cu->qp = (uint8_t)cfg->qp;
      }
      CTU_SYNC();
      const bool inside = x + cu_width <= cfg->width && y + cu_width <= cfg->height;
      if (inside) {
        const int cwim = 64 >> cfg->pu_depth_intra_max;
        const bool can_use_intra = (d >= cfg->pu_depth_intra_min && d <= cfg->pu_depth_intra_max) ||
                                   (x & ~(cwim - 1)) + cwim > cfg->width || (y & ~(cwim - 1)) + cwim > cfg->height;
        if (can_use_intra) {
          search_cu_intra(S, L, x, y, d);
          CTU_LEADER {
            if (S->best_cost < F->cost) {
              F->cost = S->best_cost;
              cur_cu->type = CU_INTRA;
              cur_cu->part_size = d > 3 ? SIZE_NxN : SIZE_2Nx2N;
              cur_cu->mode = (int8_t)S->best_mode;
            }
          }
          CTU_SYNC();
        }
        if (cur_cu->type == CU_INTRA) {
          CTU_LEADER cur_cu->mode_chroma = cur_cu->mode;
          CTU_SYNC();
          fill_cu_info(L, xl, yl, cu_width, cur_cu);
          const bool aligned = x % 8 == 0 && y % 8 == 0;
          // the references search_cu_intra built are still this CU's
          const int refs_valid = aligned ? 7 : 1;
          if (aligned && cfg->rdo >= 2 && cfg->intra_chroma_search) {
            intra_recon_cu(S, L, x, y, d, cur_cu->mode, -1, NULL, refs_valid);
            PROF_T0(PR_CHROMA);
            const int mc = search_cu_intra_chroma(S, L, x, y, d);
            PROF_ADD(S, PR_CHROMA);
            CTU_LEADER cur_cu->mode_chroma = (int8_t)mc;
            CTU_SYNC();
            fill_cu_info(L, xl, yl, cu_width, cur_cu);
            intra_recon_cu(S, L, x, y, d, -1, cur_cu->mode_chroma, NULL, 0);
          } else if (cfg->rdo >= 2) {
            // the winner's reconstruction is the one its RDO candidate computed (a leaf: depth >= 1, tr_depth == depth)
            write_back_candidate(S, L, x, y, d, cur_cu->mode, aligned);
          } else {
            // luma and chroma of the CU are independent: one pass (kvz_intra_recon_cu twice in the reference)
            intra_recon_cu(S, L, x, y, d, cur_cu->mode, aligned ? cur_cu->mode_chroma : -1, NULL, refs_valid);
          }
        }
      }
      if (cur_cu->type == CU_INTRA) {
        PROF_T0(PR_COST);
        CTU_LEADER {
          double bits = 0;
          S->sc.update = 1;
          if (cur_cu->part_size == SIZE_2Nx2N) bits += mock_encode_coding_unit(S, L, x, y, d, cur_cu);
          else bits += calc_mode_bits(S, L, cur_cu, x, y);
          double cost = bits * cfg->lambda;
          cost += cost_tr_split_accurate(S, L, xl, yl, d, cur_cu);
          F->cost = cost;
          S->sc.update = 0;
        }
        CTU_SYNC();
        PROF_ADD(S, PR_COST);
      }
      const bool can_split = cur_cu->type == CU_NOTSET || d < cfg->pu_depth_intra_max;
      CTU_LEADER {
        F->can_split = can_split;
        F->child = 0;
        F->do_children = 0;
        if (can_split) {
          F->split_cost = 0.0;
          F->cbf = cbf_is_set_any(cur_cu->cbf, d);
          F->post = S->sc;
          S->sc = F->pre;
          S->sc.update = 1;
          double split_bits = 0;
          if (d < 3) cabac_bin(&S->tb, &S->sc, CTX_SPLIT + split_model_of(L, x, y, d), 1, &split_bits);
          if (cur_cu->type == CU_INTRA && d == 3) cabac_bin(&S->tb, &S->sc, CTX_PART_SIZE, 0, &split_bits);
          S->sc.update = 0;
          F->split_cost += split_bits * cfg->lambda;
          if (cur_cu->type == CU_NOTSET || F->cbf || cfg->cu_split_termination == 1) F->do_children = 1;
          else F->split_cost = CTU_MAX_INT;
        }
        F->stage = 1;
        if (!can_split) S->ret_cost = F->cost;
      }
      CTU_SYNC();
      if (!can_split) {
        // no split possible at this depth: the CU is final, return to the parent at once
        if (d < 4) work_tree_copy_down(S, xl, yl, d);
        if (d == 0) break;
        --d;
        CTU_LEADER S->fr[d].split_cost += S->ret_cost;
        CTU_SYNC();
      }
      continue;
    }
    if (stage == 1 && descend) {
      // ---------------- children, one at a time, while the split is still cheaper
      const int k = next_child, half = cu_width / 2;
      CTU_LEADER {
        F->child = k + 1;
        S->fr[d + 1].x = x + (k & 1) * half;
        S->fr[d + 1].y = y + (k >> 1) * half;
        S->fr[d + 1].stage = 0;
      }
      CTU_SYNC();
      ++d;
      continue;
    }
    {
      // ---------------- after the children (stage 1 without a next child): combined CU, then split / no split
      CuRec *cur_cu = cu_at(L, xl, yl);
      const bool inside = x + cu_width <= cfg->width && y + cu_width <= cfg->height;
      bool combine = false;
      if (cur_cu->type == CU_NOTSET && d < 4 && inside && cfg->combine_intra_cus) {
        const CuRec *cu_d1 = cu_at(&S->lv[d + 1], xl, yl);
        combine = cu_d1->type == CU_INTRA && cu_d1->depth == d + 1;
      }
      CTU_SYNC();       // (the decision is taken by everybody before the leader rewrites the record)
      if (combine) {
        CuRec *cu_d1 = cu_at(&S->lv[d + 1], xl, yl);
        {
          CTU_LEADER {
            S->tmp = S->sc;
            S->sc = F->pre;
            F->cost = 0;
            double bits = 0;
            if (d < 3) cabac_bin(&S->tb, &S->sc, CTX_SPLIT + split_model_of(L, x, y, d), 0, &bits);
            S->best_cost = bits;
            cur_cu->mode = cu_d1->mode; cur_cu->mode_chroma = cu_d1->mode_chroma;
            cur_cu->type = CU_INTRA;
            cur_cu->part_size = SIZE_2Nx2N;
          }
          CTU_SYNC();
          fill_trdepth(L, xl, yl, d, cur_cu->tr_depth);
          fill_cu_info(L, xl, yl, cu_width, cur_cu);
          intra_recon_cu(S, L, x, y, d, cur_cu->mode, cur_cu->mode_chroma, NULL, 0);
          CTU_LEADER {
            const double mode_bits = calc_mode_bits(S, L, cur_cu, x, y) + S->best_cost;
            double cost = F->cost;
            cost += mode_bits * cfg->lambda;
            cost += cost_tr_split_accurate(S, L, xl, yl, d, cur_cu);
            F->cost = cost;
            F->post = S->sc;
            S->sc = S->tmp;
          }
          CTU_SYNC();
        }
      }
      const bool split_wins = F->split_cost < F->cost;
      CTU_SYNC();
      if (split_wins) {
        CTU_LEADER F->cost = F->split_cost;
        CTU_SYNC();
        work_tree_copy_up(S, xl, yl, d);
      } else if (d > 0) {
        CTU_LEADER S->sc = F->post;
        CTU_SYNC();
        work_tree_copy_down(S, xl, yl, d);
      }
    }
    // return to the parent
    if (d == 0) break;
    CTU_LEADER S->fr[d - 1].split_cost += F->cost;
    CTU_SYNC();
    --d;
  }
}

}  // namespace kvzctu
