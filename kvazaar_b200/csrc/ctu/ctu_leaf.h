// ctu_leaf.h -- block-level operations of the CTU search driver, written for the execution model of ctu_common.h
// (every function is called by all threads of the CTA unless it says "leader only" / "team").
//
// Reference semantics restated here (8- and 10-bit, 4:2:0, flat scaling lists):
//   intra references     src/intra.c:305-559 (kvz_intra_build_reference_any / _inner), :176-204 (smoothing)
//   intra prediction     src/intra.c:252-302 + strategies/generic/intra-generic.c:49-241
//   SATD / SAD           strategies/generic/picture-generic.c:117-340, 475-501
//   transforms           strategies/generic/dct-generic.c:255-629, src/transform.c:150-222
//   quant / dequant      strategies/generic/quant-generic.c:50-180, 298-340
//   RDOQ                 src/rdo.c:346-977
//   coefficient bits     strategies/generic/encode_coding_tree-generic.c:40-284, src/encode_coding_tree.c:63-115
#pragma once
#include "ctu_common.h"

namespace kvzctu {

#if defined(__CUDA_ARCH__)
#define CTU_ATOMIC_ADD(p, v) atomicAdd((p), (v))
#define CTU_ATOMIC_OR(p, v) atomicOr((p), (v))
#else
#define CTU_ATOMIC_ADD(p, v) (*(p) += (v))
#define CTU_ATOMIC_OR(p, v) (*(p) |= (v))
#endif

// ------------------------------------------------------------------------------------------------ work memory
// Reconstruction and levels of the RDO candidates of the CU searched last (search_cu_intra), so that the winner's are
// written back instead of computed a second time.  Luma: unit (candidate * alternatives + alternative), the alternatives
// being transform / transform skip of a 4x4 unit; chroma: unit (candidate).  Units of the CU's size, back to back.
#define CTU_RDO_CANDS 6             // search_intra_rdo: at most 3 rough-search modes (2 above depth 4) and the 3 MPMs
template <typename Pix> struct CandStore {
  Pix rec_y[CTU_RDO_CANDS * 1024], rec_c[2][CTU_RDO_CANDS * 256];
  int16_t q_y[CTU_RDO_CANDS * 1024], q_c[2][CTU_RDO_CANDS * 256];
};
template <typename Pix> struct CtuWorkT {                    // per resident CTU, global memory (L2 resident)
  LcuStore<Pix> store[5];
  CandStore<Pix> cand;
  Pix src_y[64 * 64], src_u[32 * 32], src_v[32 * 32];       // lcu->ref
  // border references from the neighbouring CTUs, index 0 = top-left corner sample (lcu->top_ref / left_ref)
  Pix top_y[100], top_u[52], top_v[52], left_y[100], left_u[52], left_v[52];
};
// The 8-bit instantiations of the types the driver's host code names (CtuWork, CtuS, FrameDev, Ctx) keep their plain
// names as aliases: 8-bit code written before the sample type became a parameter compiles unchanged.
using CtuWork = CtuWorkT<uint8_t>;

template <typename Pix> struct IntraRefs {                  // kvz_intra_references: index 0 = corner, 1..2w along the edge
  Pix top[68], left[68], ftop[68], fleft[68];
  int32_t dc;                       // DC value of the unfiltered references (modes 1)
  int32_t pad;
};

// ------------------------------------------------------------------------------------------------ teams
// A team is the group of threads that evaluates one transform unit: the whole CTA for 32x32 units, one warp for 8x8 and
// 16x16 units, half a warp for the 4x4 units of batches of 4x4 units only (several units -- colour planes, RDO
// candidates -- are then evaluated side by side, one per team; see for_tu_tasks).  A 4x4 unit has 16 coefficients: on a whole warp every data-parallel stage would leave half the
// lanes idle, and its serial sections (RDOQ's walk, the coefficient bits) run on one lane either way.  The two halves
// of a warp run the same code on different units, mostly in lockstep.  `mask`: the lanes of a warp team (tsync).
struct Team { int tid, nt, warp; unsigned mask; };
#if defined(__CUDA_ARCH__)
CTU_FN Team team_cta() { Team t = { (int)threadIdx.x, (int)blockDim.x, 0, 0xffffffffu }; return t; }
CTU_FN Team team_warp() { Team t = { (int)(threadIdx.x & 31), 32, 1, 0xffffffffu }; return t; }
CTU_FN Team team_half() { Team t = { (int)(threadIdx.x & 15), 16, 1, 0xffffu << (threadIdx.x & 16) }; return t; }
CTU_FN void tsync(const Team &t) { if (t.warp) __syncwarp(t.mask); else __syncthreads(); }
#define CTU_NWARPS ((int)(blockDim.x >> 5))
#define CTU_WARP ((int)(threadIdx.x >> 5))
#define CTU_HALF ((int)(threadIdx.x >> 4))
#else
CTU_FN Team team_cta() { Team t = { 0, 1, 0, 0 }; return t; }
CTU_FN Team team_warp() { Team t = { 0, 1, 1, 0 }; return t; }
CTU_FN Team team_half() { Team t = { 0, 1, 1, 0 }; return t; }
CTU_FN void tsync(const Team &) {}
#define CTU_NWARPS 1
#define CTU_WARP 0
#define CTU_HALF 0
#endif

// All tables the search reads, compact, in shared memory (copied from the host-built CtuTables once per CTU): the serial
// sections (cost walks, RDOQ's chain) look them up constantly, and a global-memory table costs an L2 round trip per
// dependent lookup (with 200 KB of the SM given to shared memory there is next to no L1).
struct SmTables {
  int32_t ebits[128];
  uint8_t next_mps[128], next_lps[128];
  uint16_t scan4[3][16], scan8[3][64], scan16[256], scan32[1024];     // 16x16 and 32x32 always scan diagonally
  uint8_t scan_cg[3][4][64];
  uint8_t ref_top[16][16], ref_left[16][16];
  int8_t tr4[16], tr8[64], tr16[256], tr32[1024], dst4[16];
  uint8_t sig_ctx4[16], group_idx[32], min_in_group[10];
  uint8_t pad[6];
  // not a table: the absolute levels of the coefficient group being counted, one row per half-warp, the smallest team
  // (a thread-local array indexed at run time would live in local memory, behind the 34 KB of L1 three CTAs share)
  mutable int32_t abs_scratch[8][16];
};
CTU_FN const uint16_t *sm_scan(const SmTables *t, int scan_idx, int l)      // l = log2n - 2
{
  return l == 0 ? t->scan4[scan_idx] : (l == 1 ? t->scan8[scan_idx] : (l == 2 ? t->scan16 : t->scan32));
}
CTU_FN const int8_t *sm_tr(const SmTables *t, int l) { return l == 0 ? t->tr4 : (l == 1 ? t->tr8 : (l == 2 ? t->tr16 : t->tr32)); }
// every thread of the CTA
CTU_FN void sm_tables_load(SmTables *d, const CtuTables *g)
{
  #pragma unroll 1
  for (int i = CTU_TID; i < 1024; i += CTU_NT) {
    d->scan32[i] = g->scan[0][3][i]; d->tr32[i] = g->tr[3][i];
    if (i < 256) { d->scan16[i] = g->scan[0][2][i]; d->tr16[i] = g->tr[2][i]; ((uint8_t *)d->ref_top)[i] = ((const uint8_t *)g->ref_top)[i]; ((uint8_t *)d->ref_left)[i] = ((const uint8_t *)g->ref_left)[i]; }
    if (i < 768) ((uint8_t *)d->scan_cg)[i] = ((const uint8_t *)g->scan_cg)[i];
    if (i < 192) d->scan8[i / 64][i % 64] = g->scan[i / 64][1][i % 64];
    if (i < 128) { d->ebits[i] = g->ebits[i]; d->next_mps[i] = g->next_mps[i]; d->next_lps[i] = g->next_lps[i]; }
    if (i < 64) d->tr8[i] = g->tr[1][i];
    if (i < 48) d->scan4[i / 16][i % 16] = g->scan[i / 16][0][i % 16];
    if (i < 32) d->group_idx[i] = g->group_idx[i];
    if (i < 16) { d->tr4[i] = g->tr[0][i]; d->dst4[i] = g->dst4[i]; d->sig_ctx4[i] = g->sig_ctx4[i]; }
    if (i < 10) d->min_in_group[i] = g->min_in_group[i];
  }
}

// Scratch of one transform-unit evaluation, carved out of the team's part of the arena for nn = n*n coefficients.
template <typename Pix> struct TuFixed {
  double prep_c0[16], prep_sig0[16], prep_sig1[16];
  int32_t prep_ld[16], prep_ctx_sig[16];
  int32_t last_x_bits[12], last_y_bits[12];
  uint8_t prep_flags[16];
  int32_t best_last_p1;
  int32_t has, ac_sum, ssd;
  uint32_t cg_mask[2];              // coefficient groups (raster) with a level != 0, of the unit's final levels
  uint32_t ts_mask[2];
  // transform skip decision (kvz_quantize_residual_trskip): both alternatives of a 4x4 luma unit
  Pix ts_rec[2][16];
  int16_t ts_coeff[2][16];
  int32_t ts_has[2], ts_ssd[2];
  int32_t ts_pick, pad;
};
static_assert(sizeof(TuFixed<uint8_t>) % 8 == 0 && sizeof(TuFixed<uint16_t>) % 8 == 0, "TuFixed alignment");
template <typename Pix> struct TuS {
  unsigned char *base;
  int nn, ncg;
  // doubles
  CTU_MFN double *cost_coeff() const { return (double *)base; }
  CTU_MFN double *cg_sig_cost() const { return (double *)base + nn; }
  CTU_MFN TuFixed<Pix> *fx() const { return (TuFixed<Pix> *)((double *)base + nn + ncg); }
  // 32-bit: kvz_sh_rates_t (rdo.h:49-58); d (delta_u of kvz_quant's sign hiding) shares inc: never both
  CTU_MFN int32_t *i32() const { return (int32_t *)(base + 8 * (nn + ncg) + sizeof(TuFixed<Pix>)); }
  CTU_MFN int32_t *inc() const { return i32(); }
  CTU_MFN int32_t *dec() const { return i32() + nn; }
  CTU_MFN int32_t *sig_inc() const { return i32() + 2 * nn; }
  CTU_MFN int32_t *qdelta() const { return i32() + 3 * nn; }
  CTU_MFN int32_t *d() const { return i32(); }
  CTU_MFN int32_t *cg_flag() const { return i32() + 4 * nn; }
  CTU_MFN int32_t *cg_nzflag() const { return i32() + 4 * nn + ncg; }
  // 16-bit
  CTU_MFN int16_t *i16() const { return (int16_t *)(i32() + 4 * nn + 2 * ncg); }
  CTU_MFN int16_t *a() const { return i16(); }             // residual / inverse-transform output
  CTU_MFN int16_t *b() const { return i16() + nn; }        // transform coefficients
  CTU_MFN int16_t *q() const { return i16() + 2 * nn; }    // quantised levels
  CTU_MFN int16_t *t() const { return i16() + 3 * nn; }    // intermediate of the separable passes
  CTU_MFN uint16_t *cg_nz() const { return (uint16_t *)(i16() + 4 * nn); }
  // bytes
  CTU_MFN uint8_t *u8() const { return (uint8_t *)(i16() + 4 * nn + ncg + (ncg & 1)); }
  CTU_MFN uint8_t *sig_code() const { return u8(); }
  CTU_MFN Pix *pred() const { return (Pix *)(u8() + nn); }
  CTU_MFN Pix *rec() const { return pred() + nn; }
};
template <typename Pix> CTU_FN int tu_scratch_bytes(int nn)
{
  const int ncg = nn >= 16 ? nn / 16 : 1;
  const int b = 8 * (nn + ncg) + (int)sizeof(TuFixed<Pix>) + 4 * (4 * nn + 2 * ncg) + 2 * (4 * nn + ncg + (ncg & 1)) + nn + 2 * nn * (int)sizeof(Pix);
  return (b + 15) & ~15;
}
template <typename Pix> CTU_FN TuS<Pix> tu_scratch(unsigned char *arena, int nn, int slot)
{
  TuS<Pix> t;
  t.nn = nn; t.ncg = nn >= 16 ? nn / 16 : 1;
  t.base = arena + (size_t)slot * tu_scratch_bytes<Pix>(nn);
  return t;
}
// One 32x32 unit, or four units of up to 16x16 side by side.  With 16-bit samples four 16x16 units need 42 176 bytes:
// the arena keeps its size (three CTAs per SM) and for_tu_tasks runs batches with such units one after another on the
// whole CTA.
#define CTU_ARENA_BYTES 40960

// ------------------------------------------------------------------------------------------------ pixel planes
template <typename Pix> struct Plane { Pix *rec; const Pix *src; const Pix *top; const Pix *left; int16_t *coeff; int lw; };
template <typename Pix> CTU_FN Plane<Pix> plane_of(CtuWorkT<Pix> *W, LcuLevel<Pix> *L, int color)
{
  Plane<Pix> p;
  if (color == 0) { p.rec = L->rec_y; p.src = W->src_y; p.top = W->top_y; p.left = W->left_y; p.coeff = L->coeff_y; p.lw = 64; }
  else if (color == 1) { p.rec = L->rec_u; p.src = W->src_u; p.top = W->top_u; p.left = W->left_u; p.coeff = L->coeff_u; p.lw = 32; }
  else { p.rec = L->rec_v; p.src = W->src_v; p.top = W->top_v; p.left = W->left_v; p.coeff = L->coeff_v; p.lw = 32; }
  return p;
}

// ------------------------------------------------------------------------------------------------ intra references
// kvz_intra_build_reference for the blocks of the colours in `mask` (bit per colour) at luma position (x, y) (picture
// coordinates), into r[colour], followed by the [1 2 1] smoothing (done eagerly: the reference's lazy flag only saves
// time; chroma never reads it) and the DC sum.  log2w[colour]: the block sizes.  One pass over all colours: the border
// reads of the three planes overlap instead of queueing behind each other.
template <typename Pix> CTU_FN_NOINLINE void build_refs_multi(const SmTables *T, const CtuConfig *cfg, CtuWorkT<Pix> *W, LcuLevel<Pix> *L, const int log2w[3], int mask, int x, int y, IntraRefs<Pix> *r)
{
  const int lx = x & 63, ly = y & 63;
  const bool has_left = x > 0, has_top = y > 0, inner = has_left && has_top;
  const int mid = 1 << (PixDepth<Pix>::bd - 1);       // value of unavailable references (ref: intra.c:319)
  int n_of[3], start[4];
  start[0] = 0;
  for (int col = 0; col < 3; ++col) { n_of[col] = ((mask >> col) & 1) ? 2 * (1 << log2w[col]) + 1 : 0; start[col + 1] = start[col] + 2 * n_of[col]; }
  #pragma unroll 1
  for (int it = CTU_TID; it < start[3]; it += CTU_NT) {
    const int color = it >= start[2] ? 2 : (it >= start[1] ? 1 : 0);
    const int i = it - start[color], n = n_of[color], w = (n - 1) >> 1;
    const int is_c = color != 0;
    const Plane<Pix> P = plane_of(W, L, color);
    const int px = lx >> is_c, py = ly >> is_c, lw = P.lw;
    int al = 0, at = 0;
    if (has_left) { al = T->ref_left[ly >> 2][lx >> 2] >> is_c; al = imin(al, 2 * w); al = imin(al, (cfg->height - y) >> is_c); }
    if (has_top) { at = T->ref_top[ly >> 2][lx >> 2] >> is_c; at = imin(at, 2 * w); at = imin(at, (cfg->width - x) >> is_c); }
    // the _inner variant copies in groups of four, at least one group (intra.c:486-494, 512-516)
    const int nl = inner ? imax(4, (al + 3) & ~3) : al;
    const int ntp = inner ? imax(4, (at + 3) & ~3) : at;
    // border accessors: k >= -1
#define CTU_TOP_BORDER(k) (py ? P.rec[(px + (k)) + (py - 1) * lw] : P.top[1 + px + (k)])
#define CTU_LEFT_BORDER(k) (px ? P.rec[(px - 1) + (py + (k)) * lw] : P.left[1 + py + (k)])
    const bool is_top = i >= n;
    const int e = is_top ? i - n : i;          // entry 0 = corner
    int v;
    if (e == 0) {
      if (inner) v = px ? CTU_TOP_BORDER(-1) : CTU_LEFT_BORDER(-1);
      else v = has_left ? CTU_LEFT_BORDER(0) : (has_top ? CTU_TOP_BORDER(0) : mid);      // "copy reference clockwise": left[1]
    } else if (!is_top) {
      if (has_left) v = CTU_LEFT_BORDER(imin(e - 1, nl - 1));
      else v = has_top ? CTU_TOP_BORDER(0) : mid;
    } else {
      if (has_top) v = CTU_TOP_BORDER(imin(e - 1, ntp - 1));
      else v = has_left ? CTU_LEFT_BORDER(0) : mid;
    }
#undef CTU_TOP_BORDER
#undef CTU_LEFT_BORDER
    (is_top ? r[color].top : r[color].left)[e] = (Pix)v;
  }
  CTU_SYNC();
  // smoothing of the luma references; one thread per colour sums the DC
  const int n0 = n_of[0];
  #pragma unroll 1
  for (int i = CTU_TID; i < 2 * n0 + 3; i += CTU_NT) {
    if (i >= 2 * n0) {
      const int color = i - 2 * n0;
      if ((mask >> color) & 1) {
        const int w = 1 << log2w[color];
        int s = 0;
        for (int k = 1; k <= w; ++k) s += r[color].top[k] + r[color].left[k];
        r[color].dc = (s + w) >> (log2w[color] + 1);
      }
      continue;
    }
    const bool is_top = i >= n0;
    const int e = is_top ? i - n0 : i;
    const Pix *p = is_top ? r[0].top : r[0].left;
    int v;
    if (e == 0) v = (r[0].left[1] + 2 * r[0].left[0] + r[0].top[1] + 2) >> 2;
    else if (e == n0 - 1) v = p[e];
    else v = (p[e - 1] + 2 * p[e] + p[e + 1] + 2) >> 2;
    (is_top ? r[0].ftop : r[0].fleft)[e] = (Pix)v;
  }
  CTU_SYNC();
}
template <typename Pix> CTU_FN void build_refs(const SmTables *T, const CtuConfig *cfg, CtuWorkT<Pix> *W, LcuLevel<Pix> *L, int log2w, int color, int x, int y, IntraRefs<Pix> *r)
{
  int l[3] = { log2w, log2w, log2w };
  build_refs_multi(T, cfg, W, L, l, 1 << color, x, y, r - color);
}

// ------------------------------------------------------------------------------------------------ intra prediction
template <typename Pix> CTU_FN int ang_ref(const Pix *rmain, const Pix *rside, int idx, int inv)
{
  if (idx >= -1) return rmain[idx + 1];
  const int k = -idx - 1;
  return rside[(128 + k * inv) >> 8];
}
template <typename Pix> CTU_FN int angular_px(int mode, const Pix *top, const Pix *left, int ox, int oy)
{
  const int disp_tab[9] = { 0, 2, 5, 9, 13, 17, 21, 26, 32 };
  const int inv_tab[9] = { 0, 4096, 1638, 910, 630, 482, 390, 315, 256 };
  const bool vertical = mode >= 18;
  const int mdisp = vertical ? mode - 26 : 10 - mode;
  const int adisp = iabs(mdisp);
  const int sdisp = mdisp < 0 ? -disp_tab[adisp] : disp_tab[adisp];
  const Pix *rmain = vertical ? top : left;
  const Pix *rside = vertical ? left : top;
  const int x = vertical ? ox : oy, y = vertical ? oy : ox;
  if (sdisp == 0) return rmain[x + 1];
  const int pos = (y + 1) * sdisp;
  const int di = pos >> 5, df = pos & 31;
  const int inv = inv_tab[adisp];
  const int r1 = ang_ref(rmain, rside, x + di, inv);
  if (df == 0) return r1;
  const int r2 = ang_ref(rmain, rside, x + di + 1, inv);
  return ((32 - df) * r1 + df * r2 + 16) >> 5;
}
CTU_FN bool intra_uses_filtered(int log2w, int mode, int color)
{
  if (color != 0 || mode == 1 || log2w == 2) return false;
  if (mode == 0) return true;
  const int thres = log2w == 3 ? 7 : (log2w == 4 ? 1 : 0);
  return imin(iabs(mode - 26), iabs(mode - 10)) > thres;
}
// kvz_intra_predict for one sample (filter_boundary is always true: no lossless / implicit RDPCM)
template <typename Pix> CTU_FN int intra_predict_px(const IntraRefs<Pix> *r, int log2w, int mode, int color, int x, int y)
{
  const bool f = intra_uses_filtered(log2w, mode, color);
  const Pix *t = f ? r->ftop : r->top, *l = f ? r->fleft : r->left;
  const int w = 1 << log2w;
  if (mode == 0) {
    const int hor = (w - 1 - x) * l[y + 1] + (x + 1) * t[w + 1];
    const int ver = (w - 1 - y) * t[x + 1] + (y + 1) * l[w + 1];
    return (ver + hor + w) >> (log2w + 1);
  }
  if (mode == 1) {
    const int dc = r->dc;
    if (color == 0 && log2w < 5) {
      if (x == 0 && y == 0) return (l[1] + 2 * dc + t[1] + 2) >> 2;
      if (y == 0) return (t[x + 1] + 3 * dc + 2) >> 2;
      if (x == 0) return (l[y + 1] + 3 * dc + 2) >> 2;
    }
    return dc;
  }
  int v = angular_px(mode, t, l, x, y);
  if (color == 0 && log2w < 5) {
    if (mode == 10 && y == 0) v = iclip(0, PixTraits<Pix>::max, v + ((t[x + 1] - t[0]) >> 1));
    else if (mode == 26 && x == 0) v = iclip(0, PixTraits<Pix>::max, v + ((l[y + 1] - l[0]) >> 1));
  }
  return v;
}
// prediction of a whole block into dst (row stride dst_stride)
template <typename Pix> CTU_FN_NOINLINE void predict_block(const IntraRefs<Pix> *r, int log2w, int mode, int color, Pix *dst, int dst_stride)
{
  const int w = 1 << log2w;
  #pragma unroll 1
  for (int e = CTU_TID; e < w * w; e += CTU_NT) {
    const int y = e >> log2w, x = e & (w - 1);
    dst[y * dst_stride + x] = (Pix)intra_predict_px(r, log2w, mode, color, x, y);
  }
  CTU_SYNC();
}

// ------------------------------------------------------------------------------------------------ SATD / SAD
CTU_FN int hadamard4_abs_sum(int d[16])
{
  // rows then columns; the sum of absolute transform values does not depend on the butterfly order
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const int a = d[4 * r] + d[4 * r + 1], b = d[4 * r] - d[4 * r + 1], c = d[4 * r + 2] + d[4 * r + 3], e = d[4 * r + 2] - d[4 * r + 3];
    d[4 * r] = a + c; d[4 * r + 1] = b + e; d[4 * r + 2] = a - c; d[4 * r + 3] = b - e;
  }
  int s = 0;
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    const int a = d[c] + d[4 + c], b = d[c] - d[4 + c], g = d[8 + c] + d[12 + c], e = d[8 + c] - d[12 + c];
    s += iabs(a + g) + iabs(b + e) + iabs(a - g) + iabs(b - e);
  }
  return s;
}
CTU_FN int hadamard8_abs_sum(int d[64])
{
#pragma unroll
  for (int r = 0; r < 8; ++r) {
    int *p = d + 8 * r;
    const int a0 = p[0] + p[4], a1 = p[1] + p[5], a2 = p[2] + p[6], a3 = p[3] + p[7];
    const int a4 = p[0] - p[4], a5 = p[1] - p[5], a6 = p[2] - p[6], a7 = p[3] - p[7];
    const int b0 = a0 + a2, b1 = a1 + a3, b2 = a0 - a2, b3 = a1 - a3, b4 = a4 + a6, b5 = a5 + a7, b6 = a4 - a6, b7 = a5 - a7;
    p[0] = b0 + b1; p[1] = b0 - b1; p[2] = b2 + b3; p[3] = b2 - b3; p[4] = b4 + b5; p[5] = b4 - b5; p[6] = b6 + b7; p[7] = b6 - b7;
  }
  int s = 0;
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    const int *p = d + c;
    const int a0 = p[0] + p[32], a1 = p[8] + p[40], a2 = p[16] + p[48], a3 = p[24] + p[56];
    const int a4 = p[0] - p[32], a5 = p[8] - p[40], a6 = p[16] - p[48], a7 = p[24] - p[56];
    const int b0 = a0 + a2, b1 = a1 + a3, b2 = a0 - a2, b3 = a1 - a3, b4 = a4 + a6, b5 = a5 + a7, b6 = a4 - a6, b7 = a5 - a7;
    s += iabs(b0 + b1) + iabs(b0 - b1) + iabs(b2 + b3) + iabs(b2 - b3) + iabs(b4 + b5) + iabs(b4 - b5) + iabs(b6 + b7) + iabs(b6 - b7);
  }
  return s;
}

// ---- rough search: SATD of every mode
// Angular modes are predicted from a per-mode extended main reference: entry idx + w holds what the reference's
// ref_main[idx + 1] holds (intra-generic.c:86-122) -- the main edge for idx >= -1, the projected side edge below --
// so that a sample is one branch-free two-tap interpolation.  Horizontal modes are evaluated transposed (main = left,
// block and source transposed): the SATD / SAD of a block and of its transpose are the same.
template <typename Pix> struct RoughExt { Pix e[33][104]; };      // [mode - 2][idx + w], idx in [-w, 2w + 1]
static_assert(sizeof(RoughExt<uint16_t>) <= CTU_ARENA_BYTES, "rough-search scratch lives in the arena");

CTU_FN void ang_params(int mode, bool *vertical, int *sdisp, int *inv)
{
  const int disp_tab[9] = { 0, 2, 5, 9, 13, 17, 21, 26, 32 };
  const int inv_tab[9] = { 0, 4096, 1638, 910, 630, 482, 390, 315, 256 };
  *vertical = mode >= 18;
  const int mdisp = *vertical ? mode - 26 : 10 - mode;
  const int adisp = iabs(mdisp);
  *sdisp = mdisp < 0 ? -disp_tab[adisp] : disp_tab[adisp];
  *inv = inv_tab[adisp];
}

// difference block (prediction - source) of the w8 x w8 sub-block at (bx, by) of mode m into d[], row-major, in the
// mode's own orientation (transposed for horizontal modes)
template <int W8, typename Pix>
CTU_FN void rough_diff_block(const IntraRefs<Pix> *r, const RoughExt<Pix> *ext, int log2w, int color, int m, const Pix *src, int src_stride, int bx, int by, int *d)
{
  const int w = 1 << log2w;
  if (m >= 2) {
    bool vertical; int sdisp, inv;
    ang_params(m, &vertical, &sdisp, &inv);
    const Pix *e = ext->e[m - 2] + w;
    // transposed domain of a horizontal mode: row index <-> picture column
    const int ox = vertical ? bx : by, oy = vertical ? by : bx;
    const int sx = vertical ? 1 : src_stride, sy = vertical ? src_stride : 1;
    const bool f = intra_uses_filtered(log2w, m, color);
    const Pix *side = vertical ? (f ? r->fleft : r->left) : (f ? r->ftop : r->top);
    const bool edge = color == 0 && log2w < 5 && sdisp == 0 && ox == 0;      // modes 10 / 26: first column filtered
#pragma unroll
    for (int y = 0; y < W8; ++y) {
      const int pos = (oy + y + 1) * sdisp;
      const int di = pos >> 5, df = pos & 31;
      const Pix *p = e + ox + di;
#pragma unroll
      for (int x = 0; x < W8; ++x) {
        int v = ((32 - df) * (int)p[x] + df * (int)p[x + 1] + 16) >> 5;
        if (edge && x == 0) v = iclip(0, PixTraits<Pix>::max, v + (((int)side[oy + y + 1] - (int)side[0]) >> 1));
        d[y * W8 + x] = v - (int)src[(oy + y) * sy + (ox + x) * sx];
      }
    }
  } else {
    // planar (filtered references for luma blocks above 4x4) and DC (unfiltered, edge-filtered for luma below 32x32)
    const bool f = intra_uses_filtered(log2w, m, color);
    const Pix *t = f ? r->ftop : r->top, *l = f ? r->fleft : r->left;
    const int tr = t[w + 1], bl = l[w + 1], dc = r->dc;
    const bool dc_edges = color == 0 && log2w < 5;
#pragma unroll
    for (int y = 0; y < W8; ++y) {
      const int yy = by + y, ly = l[yy + 1];
#pragma unroll
      for (int x = 0; x < W8; ++x) {
        const int xx = bx + x;
        int v;
        if (m == 0) v = ((w - 1 - xx) * ly + (xx + 1) * tr + (w - 1 - yy) * (int)t[xx + 1] + (yy + 1) * bl + w) >> (log2w + 1);
        else {
          v = dc;
          if (dc_edges) {
            if (xx == 0 && yy == 0) v = (ly + 2 * dc + (int)t[1] + 2) >> 2;
            else if (yy == 0) v = ((int)t[xx + 1] + 3 * dc + 2) >> 2;
            else if (xx == 0) v = (ly + 3 * dc + 2) >> 2;
          }
        }
        d[y * W8 + x] = v - (int)src[yy * src_stride + xx];
      }
    }
  }
}

// SATD (satd_NxN) and, for 4x4, SAD of the prediction of every mode against the source block.
// satd_out / sad_out: [35] ints.  `ext`: scratch (the arena: no transform-unit job is running during the rough search).
template <typename Pix> CTU_FN_NOINLINE void rough_costs_all_modes(const IntraRefs<Pix> *r, RoughExt<Pix> *ext, int log2w, int color, const Pix *src, int src_stride,
                                  int32_t *satd_out, int32_t *sad_out, bool want_sad)
{
  const int w = 1 << log2w;
  #pragma unroll 1
  for (int m = CTU_TID; m < 35; m += CTU_NT) { satd_out[m] = 0; sad_out[m] = 0; }
  // extended main references of the 33 angular modes
  const int len = 3 * w + 2;
  #pragma unroll 1
  for (int it = CTU_TID; it < 33 * len; it += CTU_NT) {
    const int m = 2 + it / len, idx = it % len - w;
    bool vertical; int sdisp, inv;
    ang_params(m, &vertical, &sdisp, &inv);
    const bool f = intra_uses_filtered(log2w, m, color);
    const Pix *t = f ? r->ftop : r->top, *l = f ? r->fleft : r->left;
    const Pix *rmain = vertical ? t : l, *rside = vertical ? l : t;
    int v = 0;
    if (idx >= -1) { if (idx + 1 <= 2 * w) v = rmain[idx + 1]; }
    else if (sdisp < 0) v = rside[(128 + (-idx - 1) * inv) >> 8];
    ext->e[m - 2][idx + w] = (Pix)v;
  }
  CTU_SYNC();
  if (w == 4) {
    #pragma unroll 1
    for (int m = CTU_TID; m < 35; m += CTU_NT) {
      int d[16], sad = 0;
      rough_diff_block<4>(r, ext, 2, color, m, src, src_stride, 0, 0, d);
#pragma unroll
      for (int e = 0; e < 16; ++e) sad += iabs(d[e]);
      satd_out[m] = (hadamard4_abs_sum(d) + 1) >> 1;
      if (want_sad) sad_out[m] = sad;
    }
  } else {
    const int sb = w >> 3, nsb = sb * sb, items = 35 * nsb;
    #pragma unroll 1
    for (int it = CTU_TID; it < items; it += CTU_NT) {
      const int m = it / nsb, k = it % nsb, bx = (k % sb) * 8, by = (k / sb) * 8;
      int d[64];
      rough_diff_block<8>(r, ext, log2w, color, m, src, src_stride, bx, by, d);
      CTU_ATOMIC_ADD(&satd_out[m], (hadamard8_abs_sum(d) + 2) >> 2);
    }
  }
  CTU_SYNC();
  if constexpr (PixDepth<Pix>::bd != 8) {
    // above 8 bits the reference's SATD of 8x8 and larger blocks and its SAD are scaled to 8-bit precision
    // (strategies-picture.h:68, picture-generic.c:381, 484, 521); the 4x4 SATD is not
    constexpr int sh = PixDepth<Pix>::bd - 8;
    #pragma unroll 1
    for (int m = CTU_TID; m < 35; m += CTU_NT) { if (w > 4) satd_out[m] >>= sh; sad_out[m] >>= sh; }
    CTU_SYNC();
  }
}

// kvz_pixels_calc_ssd over a w x w block (result in *out after the call; out must be zeroed by the leader before)
template <typename Pix> CTU_FN_NOINLINE void ssd_block(const Pix *a, int sa, const Pix *b, int sb, int w, int32_t *out)
{
  int acc = 0;
  #pragma unroll 1
  for (int e = CTU_TID; e < w * w; e += CTU_NT) {
    const int y = e / w, x = e - y * w;
    const int d = (int)a[y * sa + x] - (int)b[y * sb + x];
    acc += d * d;
  }
  if (acc) CTU_ATOMIC_ADD(out, acc);
  CTU_SYNC();
}

// ------------------------------------------------------------------------------------------------ transforms
// two int16 x int8 products per instruction (IDP2A); the pairs must be 4-byte (samples) / 2-byte (matrix) aligned
#if defined(__CUDA_ARCH__)
CTU_FN int dot4_s16_s8(const int16_t *s, const int8_t *m, int acc)
{
  const int2 sv = *reinterpret_cast<const int2 *>(s);       // 4 samples
  const int mv = *reinterpret_cast<const int *>(m);         // 4 matrix bytes
  acc = __dp2a_lo(sv.x, mv, acc);
  return __dp2a_hi(sv.y, mv, acc);
}
#else
CTU_FN int dot4_s16_s8(const int16_t *s, const int8_t *m, int acc) { return acc + s[0] * m[0] + s[1] * m[1] + s[2] * m[2] + s[3] * m[3]; }
#endif

// forward: dst[k*N + j] = (int16)((sum_i M[k][i] * src[j*N + i] + add) >> shift)
// L2N != 0: the size is a compile-time constant (the 4x4 path: most transform units of a CTU)
template <int L2N>
CTU_FN_NOINLINE void fwd_pass(const Team &tm, const int16_t *src, int16_t *dst, const int8_t *M, int n_rt, int shift)
{
  const int add = 1 << (shift - 1);
  const int n = L2N ? (1 << L2N) : n_rt;
  const int log2n = L2N ? L2N : (n == 4 ? 2 : (n == 8 ? 3 : (n == 16 ? 4 : 5)));
  #pragma unroll 1
  for (int e = tm.tid; e < n * n; e += tm.nt) {
    const int k = e >> log2n, j = e & (n - 1);
    const int16_t *s = src + (j << log2n);
    const int8_t *m = M + (k << log2n);
    int acc = 0;
    for (int i = 0; i < n; i += 4) acc = dot4_s16_s8(s + i, m + i, acc);
    dst[e] = (int16_t)((acc + add) >> shift);
  }
  tsync(tm);
}
// inverse: dst[j*N + k] = clip16((sum_i M[i][k] * src[i*N + j] + add) >> shift)
template <int L2N>
CTU_FN_NOINLINE void inv_pass(const Team &tm, const int16_t *src, int16_t *dst, const int8_t *M, int n_rt, int shift)
{
  const int add = 1 << (shift - 1);
  const int n = L2N ? (1 << L2N) : n_rt;
  const int log2n = L2N ? L2N : (n == 4 ? 2 : (n == 8 ? 3 : (n == 16 ? 4 : 5)));
  #pragma unroll 1
  for (int e = tm.tid; e < n * n; e += tm.nt) {
    const int j = e >> log2n, k = e & (n - 1);
    const int8_t *m = M + k;
    const int16_t *sp = src + j;
    int acc = 0;
#pragma unroll 4
    for (int i = 0; i < n; ++i) acc += (int)m[i << log2n] * (int)sp[i << log2n];
    dst[e] = (int16_t)iclip(-32768, 32767, (acc + add) >> shift);
  }
  tsync(tm);
}

CTU_FN int ilog2(int n) { int l = 0; while ((1 << l) < n) ++l; return l; }

// ------------------------------------------------------------------------------------------------ quantisation
CTU_FN int quant_scale(int r) { const int t[6] = { 26214, 23302, 20560, 18396, 16384, 14564 }; return t[r]; }
CTU_FN int inv_quant_scale(int r) { const int t[6] = { 40, 45, 51, 57, 64, 72 }; return t[r]; }

// sign-bit hiding of kvz_quant for one coefficient group (ref: quant-generic.c:84-176)
CTU_FN void quant_sign_hide_group(const SmTables *T, const int16_t *coef, int16_t *q, const int32_t *delta_u, const int32_t *cg_nz,
                                  int num_cg, int g, int scan_idx, int log2n)
{
  bool last_cg = true;
  for (int h = g + 1; h < num_cg; ++h) if (cg_nz[h]) { last_cg = false; break; }
  const uint16_t *pos = &sm_scan(T, scan_idx, log2n - 2)[g * 16];
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

// kvz_quant: b -> q (intra slice: rounding offset 171)
template <typename Pix> CTU_FN_NOINLINE void quant_block(const Team &tm, const SmTables *T, const CtuConfig *cfg, const TuS<Pix> &tu, int n, int type, int scan_idx)
{
  const int log2n = ilog2(n);
  const int qp_scaled = scaled_qp_px<Pix>(type, cfg->qp);
  const int qc = quant_scale(qp_scaled % 6);
  const int transform_shift = 15 - PixDepth<Pix>::bd - log2n;
  const int q_bits = 14 + qp_scaled / 6 + transform_shift;
  const int add = 171 << (q_bits - 9);
  const int q_bits8 = q_bits - 8;
  int16_t *b = tu.b(), *q = tu.q();
  int32_t *d = tu.d();
  TuFixed<Pix> *fx = tu.fx();
  if (tm.tid == 0) fx->ac_sum = 0;
  tsync(tm);
  int ac = 0;
  #pragma unroll 1
  for (int e = tm.tid; e < n * n; e += tm.nt) {
    const int level_in = b[e];
    const long long abs_level = iabs(level_in);
    int level = (int)((abs_level * qc + add) >> q_bits);
    ac += level;
    d[e] = (int)((abs_level * qc - ((long long)level << q_bits)) >> q_bits8);
    level = level_in < 0 ? -level : level;
    q[e] = (int16_t)iclip(-32768, 32767, level);
  }
  if (ac) CTU_ATOMIC_ADD(&fx->ac_sum, ac);
  tsync(tm);
  if (!cfg->signhide_enable || fx->ac_sum < 2) return;
  const int num_cg = (n * n) >> 4;
  int32_t *cg_nz = tu.cg_nzflag();
  #pragma unroll 1
  for (int g = tm.tid; g < num_cg; g += tm.nt) {
    int nz = 0;
    for (int k = 0; k < 16; ++k) nz |= q[sm_scan(T, scan_idx, log2n - 2)[g * 16 + k]] != 0;
    cg_nz[g] = nz;
  }
  tsync(tm);
  #pragma unroll 1
  for (int g = tm.tid; g < num_cg; g += tm.nt)
    if (cg_nz[g]) quant_sign_hide_group(T, b, q, d, cg_nz, num_cg, g, scan_idx, log2n);
  tsync(tm);
}

// kvz_dequant: q -> b.  type: 0 luma, 2 / 3 chroma
template <int L2N, typename Pix>
CTU_FN_NOINLINE void dequant_block(const Team &tm, const CtuConfig *cfg, const TuS<Pix> &tu, int n_rt, int type)
{
  const int n = L2N ? (1 << L2N) : n_rt;
  const int transform_shift = 15 - PixDepth<Pix>::bd - (L2N ? L2N : ilog2(n));
  const int qp_scaled = scaled_qp_px<Pix>(type, cfg->qp);
  const int shift = 20 - 14 - transform_shift;
  const int scale = inv_quant_scale(qp_scaled % 6) << (qp_scaled / 6);
  const int add = 1 << (shift - 1);
  int16_t *b = tu.b();
  const int16_t *q = tu.q();
  #pragma unroll 1
  for (int e = tm.tid; e < n * n; e += tm.nt)
    b[e] = (int16_t)iclip(-32768, 32767, ((int)q[e] * scale + add) >> shift);
  tsync(tm);
}

// ------------------------------------------------------------------------------------------------ RDOQ
#define CTU_RDOQ_ONE_BIT (1 << 15)
struct RdoqModels { const uint8_t *sig, *one, *abs, *cg, *last_x, *last_y, *cbf; const int32_t *eb; uint8_t root_cbf; };
#define rq_ebits(st, bin) (m.eb[(st) ^ (bin)])

CTU_FN int rdoq_level_rate(const RdoqModels &m, uint32_t abs_level, int ctx_one, int ctx_abs, int rice, uint32_t c1_idx, uint32_t c2_idx)
{
  int rate = CTU_RDOQ_ONE_BIT;
  const uint32_t base_level = (c1_idx < 8) ? (2 + (c2_idx < 1)) : 1;
  if (abs_level >= base_level) {
    int symbol = (int)(abs_level - base_level);
    if (symbol < (3 << rice)) {
      rate += ((symbol >> rice) + 1 + rice) * CTU_RDOQ_ONE_BIT;
    } else {
      int length = rice;
      symbol -= 3 << rice;
      while (symbol >= (1 << length)) symbol -= 1 << (length++);
      rate += (3 + length + 1 - rice + length) * CTU_RDOQ_ONE_BIT;
    }
    if (c1_idx < 8) {
      rate += rq_ebits(m.one[ctx_one], 1);
      if (c2_idx < 1) rate += rq_ebits(m.abs[ctx_abs], 1);
    }
  } else if (abs_level == 1) {
    rate += rq_ebits(m.one[ctx_one], 0);
  } else if (abs_level == 2) {
    rate += rq_ebits(m.one[ctx_one], 1);
    rate += rq_ebits(m.abs[ctx_abs], 0);
  }
  return rate;
}

// context increment of sig_coeff_flag (ref: context.c:366-397)
CTU_FN int sig_ctx_inc(const SmTables *T, int pattern, int scan_idx, int px, int py, int log2n, int type)
{
  if (px + py == 0) return 0;
  if (log2n == 2) return T->sig_ctx4[4 * py + px];
  const int offset = (log2n == 3) ? (scan_idx == 0 ? 9 : 15) : (type == 0 ? 21 : 12);
  const int sx = px & 3, sy = py & 3;
  int cnt;
  if (pattern == 0) cnt = (sx + sy <= 2) ? ((sx + sy == 0) ? 2 : 1) : 0;
  else if (pattern == 1) cnt = (sy <= 1) ? ((sy == 0) ? 2 : 1) : 0;
  else if (pattern == 2) cnt = (sx <= 1) ? ((sx == 0) ? 2 : 1) : 0;
  else cnt = 2;
  return ((type == 0 && ((px >> 2) + (py >> 2)) > 0) ? 3 : 0) + offset + cnt;
}

// kvz_rdoq_sign_hiding (ref: rdo.c:518-653); serial, one thread
template <typename Pix> CTU_FN_NOINLINE void rdoq_sign_hiding(const TuS<Pix> &tu, const uint16_t *blk, double lambda, int qp_scaled, int last_pos, const int16_t *coef, int16_t *q)
{
  const int32_t *s_inc = tu.inc(), *s_dec = tu.dec(), *s_sig_inc = tu.sig_inc(), *s_qdelta = tu.qdelta();
  const int inv_quant = inv_quant_scale(qp_scaled % 6);
  const long long rd_factor = (long long)(inv_quant * inv_quant * (1 << (2 * (qp_scaled / 6))) / lambda / 16 / (1 << (2 * (PixDepth<Pix>::bd - 8))) + 0.5);
  const int last_cg = (last_pos - 1) >> 4;
  for (int cg = last_cg; cg >= 0; --cg) {
    const uint16_t *pos = blk + (cg << 4);
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
        if (a == 1) dec_bits -= CTU_RDOQ_ONE_BIT + s_sig_inc[p];
        if (cg == last_cg && last_nz == k && a == 1) dec_bits -= 4 * CTU_RDOQ_ONE_BIT;
        inc_bits = -quant_cost + inc_bits;
        dec_bits = quant_cost + dec_bits;
        if (inc_bits < dec_bits) { change = 1; cost = inc_bits; }
        else {
          change = -1; cost = dec_bits;
          if (k == first_nz && a == 1) cost = 0x7FFFFFFFFFFFFFFFLL;
        }
      } else {
        const int bits = CTU_RDOQ_ONE_BIT + s_inc[p] + s_sig_inc[p];
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

// RDOQ runs on the first nl = rdoq_lanes() threads of a team (the first warp of a CTA team), whose lanes are `mask`
CTU_FN int rdoq_lanes(const Team &t) { return t.nt < CTU_TEAM_N ? t.nt : CTU_TEAM_N; }
#if defined(__CUDA_ARCH__)
CTU_FN void rq_sync(unsigned mask) { __syncwarp(mask); }
CTU_FN int team_max(int v, unsigned mask, int nl) { for (int o = nl >> 1; o > 0; o >>= 1) v = max(v, __shfl_xor_sync(mask, v, o)); return v; }
CTU_FN int team_sum(int v, unsigned mask, int nl) { for (int o = nl >> 1; o > 0; o >>= 1) v += __shfl_xor_sync(mask, v, o); return v; }
#else
CTU_FN void rq_sync(unsigned) {}
CTU_FN int team_max(int v, unsigned, int) { return v; }
CTU_FN int team_sum(int v, unsigned, int) { return v; }
#endif

// kvz_rdoq for one TU, executed by the RDOQ lanes of a team (lane < nl): coef = tu->b, levels to tu->q.  `cabac` = the
// models of state->cabac (NOT the search copy: rdo.c:665).  type 0 luma / 2 chroma; tr_depth as in quant-generic.c:237-238.
template <int L2N, typename Pix>
CTU_FN_NOINLINE void rdoq_team(const SmTables *T, const SmTables *tb, const CtuConfig *cfg, const uint8_t *cabac, const TuS<Pix> &tu, int log2n_rt, int type,
                      int scan_idx, int tr_depth, int lane, int nl, unsigned mask)
{
  const int log2n = L2N ? L2N : log2n_rt;
  const int16_t *coef = tu.b();
  int16_t *q = tu.q();
  TuFixed<Pix> &s = *tu.fx();
  double *s_cost_coeff = tu.cost_coeff(), *s_cg_sig_cost = tu.cg_sig_cost();
  uint8_t *s_sig_code = tu.sig_code();
  int32_t *s_inc = tu.inc(), *s_dec = tu.dec(), *s_sig_inc = tu.sig_inc(), *s_qdelta = tu.qdelta(), *s_cg_flag = tu.cg_flag();
  uint16_t *s_cg_nz = tu.cg_nz();
  const int n = 1 << log2n, nn = n * n;
  const int transform_shift = 15 - PixDepth<Pix>::bd - log2n;
  const int qp_scaled = scaled_qp_px<Pix>(type, cfg->qp);
  const int q_bits = 14 + qp_scaled / 6 + transform_shift;
  const int qc = quant_scale(qp_scaled % 6);
  const int half = 1 << (q_bits - 1);
  const double lambda = cfg->lambda;
  const bool SH = cfg->signhide_enable != 0;
  // error scale (scalinglist.c:351-368): 2^15 * 2^(-2 * transform_shift) / q / q / 2^(2 * (bd - 8))
  double err_scale = 32768.0;
  for (int i = 0; i < 2 * transform_shift; ++i) err_scale *= 0.5;
  for (int i = 0; i > 2 * transform_shift; --i) err_scale *= 2.0;
  err_scale = err_scale / qc / qc / (1 << (2 * (PixDepth<Pix>::bd - 8)));
  RdoqModels m;
  m.eb = tb->ebits;
  m.sig = cabac + (type ? CTX_SIG_CHROMA : CTX_SIG_LUMA);
  m.one = cabac + (type ? CTX_ONE_CHROMA : CTX_ONE_LUMA);
  m.abs = cabac + (type ? CTX_ABS_CHROMA : CTX_ABS_LUMA);
  m.cg = cabac + CTX_SIG_CG + type;
  m.last_x = cabac + (type ? CTX_LAST_X_CHROMA : CTX_LAST_X_LUMA);
  m.last_y = cabac + (type ? CTX_LAST_Y_CHROMA : CTX_LAST_Y_LUMA);
  m.cbf = cabac + (type ? CTX_CBF_CHROMA : CTX_CBF_LUMA);
  m.root_cbf = cabac[CTX_ROOT_CBF];
  auto sig_cost_of = [&](uint8_t code) { return (code >> 6) == 2 ? 0.0 : lambda * rq_ebits(m.sig[code & 63], code >> 6); };
  auto level0_cost = [&](int blk) { const double e = (double)imin(iabs((int)coef[blk]) * qc, 0x7FFFFFFF - half); return e * e * err_scale; };
  const uint16_t *blk_of = sm_scan(T, scan_idx, log2n - 2);

  int my_last = -1;
  #pragma unroll 1
  for (int sp = lane; sp < nn; sp += nl) {
    const int ld = imin(iabs((int)coef[blk_of[sp]]) * qc, 0x7FFFFFFF - half);
    if (((ld + half) >> q_bits) > 0) my_last = sp;
  }
  const int last_scanpos = team_max(my_last, mask, nl);
  rq_sync(mask);
  #pragma unroll 1
  for (int sp = lane; sp < nn; sp += nl) if (sp > last_scanpos) q[blk_of[sp]] = 0;
  if (last_scanpos < 0) { rq_sync(mask); return; }
  #pragma unroll 1
  for (int g = lane; g < nn / 16; g += nl) { s_cg_flag[g] = 0; s_cg_sig_cost[g] = 0; }
  if (lane == 0) {
    if (SH) s_sig_inc[blk_of[last_scanpos]] = 0;
    const int cb = log2n - 2;
    const int off = type ? 0 : (cb * 3 + ((cb + 1) >> 2));
    const int sh = type ? cb : ((cb + 3) >> 2);
    int bx = 0, by = 0, ctx;
    const int groups = T->group_idx[n - 1];
    for (ctx = 0; ctx < groups; ++ctx) {
      const int o = off + (ctx >> sh);
      s.last_x_bits[ctx] = bx + rq_ebits(m.last_x[o], 0); bx += rq_ebits(m.last_x[o], 1);
      s.last_y_bits[ctx] = by + rq_ebits(m.last_y[o], 0); by += rq_ebits(m.last_y[o], 1);
    }
    s.last_x_bits[ctx] = bx; s.last_y_bits[ctx] = by;
  }
  rq_sync(mask);

  const int cg_last = last_scanpos >> 4;
  const int cgs_side = n >> 2;
  int ctx_set = (last_scanpos > 0 && type == 0) ? 2 : 0;
  int c1 = 1, c2 = 0, rice = 0;
  uint32_t c1_idx = 0, c2_idx = 0;
  double base_cost = 0, block_uncoded_cost = 0;

  for (int cg = cg_last; cg >= 0; --cg) {
    const int cg_first = blk_of[cg << 4];
    const int cgx = (cg_first & (n - 1)) >> 2, cgy = (cg_first >> log2n) >> 2;
    const int cg_blk = cgy * cgs_side + cgx;
    const int right = (cgx < cgs_side - 1) ? (s_cg_flag[cgy * cgs_side + cgx + 1] != 0) : 0;
    const int lower = (cgy < cgs_side - 1) ? (s_cg_flag[(cgy + 1) * cgs_side + cgx] != 0) : 0;
    const int pattern = (n == 4) ? -1 : right + (lower << 1);
    #pragma unroll 1
    for (int k = lane; k < 16; k += nl) {
      const int sp = (cg << 4) + k;
      uint8_t fl = 0;
      if (sp <= last_scanpos) {
        fl = 1;
        const int blk = blk_of[sp];
        const int ld = imin(iabs((int)coef[blk]) * qc, 0x7FFFFFFF - half);
        const double err = (double)ld;
        const double c0 = err * err * err_scale;
        s.prep_ld[k] = ld;
        s.prep_c0[k] = c0;
        const bool cand = sp == last_scanpos || ((ld + half) >> q_bits) != 0;
        if (cand) fl |= 2;
        if (sp != last_scanpos) {
          const int ctx_sig = sig_ctx_inc(T, pattern, scan_idx, blk & (n - 1), blk >> log2n, log2n, type);
          const double sig0 = lambda * rq_ebits(m.sig[ctx_sig], 0);
          s.prep_sig0[k] = sig0;
          s.prep_sig1[k] = lambda * rq_ebits(m.sig[ctx_sig], 1);
          if (SH) s_sig_inc[blk] = rq_ebits(m.sig[ctx_sig], 1) - rq_ebits(m.sig[ctx_sig], 0);
          s.prep_ctx_sig[k] = ctx_sig;
          if (!cand) {
            s_sig_code[sp] = (uint8_t)ctx_sig; s_cost_coeff[sp] = c0 + sig0;
            q[blk] = 0;
            if (SH) s_qdelta[blk] = ld >> (q_bits - 8);
          }
        }
      }
      s.prep_flags[k] = fl;
    }
    rq_sync(mask);

    if (lane == 0) {
      double st_coded = 0, st_uncoded = 0, st_sig = 0, st_sig0 = 0;
      int nnz_before_pos0 = 0;
      unsigned nz_mask = 0;
      for (int k = 15; k >= 0; --k) {
        const uint8_t fl = s.prep_flags[k];
        if (!(fl & 1)) continue;
        const int sp = (cg << 4) + k;
        const double c0 = s.prep_c0[k], sig0k = s.prep_sig0[k];
        block_uncoded_cost += c0;
        if (!(fl & 2)) {
          const double cs = sig0k;
          base_cost += c0 + cs;
          st_sig += cs;
          if (k == 0) st_sig0 = cs;
          if (SH) s_inc[blk_of[sp]] = rq_ebits(m.one[4 * ctx_set + c1], 0);
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
        s_cost_coeff[sp] = cc;
        s_sig_code[sp] = (uint8_t)((last ? 0 : s.prep_ctx_sig[k]) | (cs_kind << 6));
        if (SH) {
          s_qdelta[blk] = (ld - (int)level * (1 << q_bits)) >> (q_bits - 8);
          if (level > 0) {
            const int now = rdoq_level_rate(m, level, one_ctx, abs_ctx, rice, c1_idx, c2_idx);
            s_inc[blk] = rdoq_level_rate(m, level + 1, one_ctx, abs_ctx, rice, c1_idx, c2_idx) - now;
            s_dec[blk] = rdoq_level_rate(m, level - 1, one_ctx, abs_ctx, rice, c1_idx, c2_idx) - now;
          } else {
            s_inc[blk] = rq_ebits(m.one[one_ctx], 0);
          }
        }
        q[blk] = (int16_t)level;
        base_cost += cc;

        const uint32_t base_level = (c1_idx < 8) ? (2 + (c2_idx < 1)) : 1;
        if (level >= base_level && level > (uint32_t)(3 * (1 << rice))) rice = imin(rice + 1, 4);
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
          nz_mask |= 1u << k;
          s_cg_flag[cg_blk] = 1;
          st_coded += cc - cs;
          st_uncoded += c0;
          if (k != 0) ++nnz_before_pos0;
        }
      }

      if (cg) {
        const int ctx_cg = right || lower;
        if (s_cg_flag[cg_blk] == 0) {
          s_cg_sig_cost[cg] = lambda * rq_ebits(m.cg[ctx_cg], 0);
          base_cost += s_cg_sig_cost[cg] - st_sig;
        } else if (cg < cg_last) {
          if (nnz_before_pos0 == 0) { base_cost -= st_sig0; st_sig -= st_sig0; }
          double cost_zero_cg = base_cost;
          s_cg_sig_cost[cg] = lambda * rq_ebits(m.cg[ctx_cg], 1);
          base_cost += s_cg_sig_cost[cg];
          cost_zero_cg += lambda * rq_ebits(m.cg[ctx_cg], 0);
          cost_zero_cg += st_uncoded;
          cost_zero_cg -= st_coded;
          cost_zero_cg -= st_sig;
          if (cost_zero_cg < base_cost) {
            nz_mask = 0;
            s_cg_flag[cg_blk] = 0;
            base_cost = cost_zero_cg;
            s_cg_sig_cost[cg] = lambda * rq_ebits(m.cg[ctx_cg], 0);
            for (int k = 15; k >= 0; --k) {
              const int sp = (cg << 4) + k, blk = blk_of[sp];
              if (q[blk]) { q[blk] = 0; s_cost_coeff[sp] = level0_cost(blk); s_sig_code[sp] = 2 << 6; }
            }
          }
        }
      } else {
        s_cg_flag[cg_blk] = 1;
      }
      s_cg_nz[cg] = (uint16_t)nz_mask;
    }
    rq_sync(mask);
  }

  if (lane == 0) {
    // best last position (rdo.c:884-945); block_type is CU_INTRA
    double best_cost;
    {
      const int ctx_cbf = type ? tr_depth : !tr_depth;
      best_cost = block_uncoded_cost + lambda * rq_ebits(m.cbf[ctx_cbf], 0);
      base_cost += lambda * rq_ebits(m.cbf[ctx_cbf], 1);
    }
    int best_last_p1 = 0;
    bool found_last = false;
    for (int cg = cg_last; cg >= 0 && !found_last; --cg) {
      const int cg_first = blk_of[cg << 4];
      const int cg_blk = ((cg_first >> log2n) >> 2) * cgs_side + ((cg_first & (n - 1)) >> 2);
      base_cost -= s_cg_sig_cost[cg];
      if (!s_cg_flag[cg_blk]) continue;
      const unsigned nz = s_cg_nz[cg];
      const int top = cg == cg_last ? (last_scanpos & 15) : 15;
      for (int k = top; k >= 0; --k) {
        const int sp = (cg << 4) + k;
        const double csk = sig_cost_of(s_sig_code[sp]);
        if (!((nz >> k) & 1)) { base_cost -= csk; continue; }
        const int blk = blk_of[sp];
        const int py = blk >> log2n, px = blk & (n - 1);
        const int gx = T->group_idx[scan_idx == 2 ? py : px], gy = T->group_idx[scan_idx == 2 ? px : py];
        double bits = s.last_x_bits[gx] + s.last_y_bits[gy];
        if (gx > 3) bits += CTU_RDOQ_ONE_BIT * ((gx - 2) >> 1);
        if (gy > 3) bits += CTU_RDOQ_ONE_BIT * ((gy - 2) >> 1);
        const double total = base_cost + lambda * bits - csk;
        if (total < best_cost) { best_last_p1 = sp + 1; best_cost = total; }
        if (q[blk] > 1) { found_last = true; break; }
        base_cost -= s_cost_coeff[sp];
        base_cost += level0_cost(blk);
      }
    }
    s.best_last_p1 = best_last_p1;
  }
  rq_sync(mask);

  const int best_last_p1 = s.best_last_p1;
  int abs_sum = 0;
  #pragma unroll 1
  for (int sp = lane; sp <= last_scanpos; sp += nl) {
    const int blk = blk_of[sp];
    if (sp < best_last_p1) {
      const int level = q[blk];
      abs_sum += level;
      q[blk] = (int16_t)(coef[blk] < 0 ? -level : level);
    } else {
      q[blk] = 0;
    }
  }
  if (SH) {
    abs_sum = team_sum(abs_sum, mask, nl);
    rq_sync(mask);
    if (lane == 0 && abs_sum >= 2) rdoq_sign_hiding(tu, blk_of, lambda, qp_scaled, best_last_p1, coef, q);
  }
  rq_sync(mask);
}

// ------------------------------------------------------------------------------------------------ CABAC bins (leader only)
// CABAC_FBITS_UPDATE with only_count = 1 (ref: cabac.h:133-139): the bit estimate of the model's current state is
// added first, then the model adapts when cabac->update is set.
CTU_FN void cabac_bin(const SmTables *tb, CabacState *c, int off, int val, double *bits)
{
  const uint8_t st = c->ctx[off];
  *bits += (double)tb->ebits[st ^ val] * (1.0 / 32768.0);
  if (c->update) c->ctx[off] = ((st & 1) == val) ? tb->next_mps[st] : tb->next_lps[st];
}

// the same with an integer accumulator in units of 2^-15 bit
CTU_FN void cabac_bin_i(const SmTables *tb, CabacState *c, int off, int val, long long *bits)
{
  const uint8_t st = c->ctx[off];
  *bits += tb->ebits[st ^ val];
  if (c->update) c->ctx[off] = ((st & 1) == val) ? tb->next_mps[st] : tb->next_lps[st];
}

CTU_FN int coeff_remain_bits(int symbol, int rice)
{
  if (symbol < (3 << rice)) return (symbol >> rice) + 1 + rice;
  int length = rice;
  symbol -= 3 << rice;
  while (symbol >= (1 << length)) { symbol -= 1 << length; ++length; }
  return 3 + length + 1 - rice + length;
}

// kvz_get_coeff_cost's CABAC branch = kvz_encode_coeff_nxn in counting mode on a copy of the search models that is
// kept when `update` is set (ref: rdo.c:223-264).  Leader only.  The cost estimate codes tr_skip as 0 (rdo.c:251-258);
// the tracker of the real coder's models passes the TU's flag.
#define CTU_NO_MASK 0xFFFFFFFFFFFFFFFFull       // (no unit has all 64 groups... a full 32x32 unit does: then the scan below is harmless)
CTU_FN_NOINLINE double coeff_cost_serial(const SmTables *T, const SmTables *tb, const CtuConfig *cfg, CabacState *c, const int16_t *coeff, int log2n, int type, int scan_idx, int tr_skip,
                                         uint64_t known_cg_mask = CTU_NO_MASK)
{
  const int n = 1 << log2n, side = n >> 2, ncg = side * side;
  uint64_t cg_flags = 0;
  if (known_cg_mask != CTU_NO_MASK) cg_flags = known_cg_mask;
  else for (int g = 0; g < ncg; ++g) {
    const int gy = g / side, gx = g - gy * side;
    bool any = false;
    for (int r = 0; r < 4 && !any; ++r) {
      const int16_t *row = coeff + (gy * 4 + r) * n + gx * 4;
      any = (row[0] | row[1] | row[2] | row[3]) != 0;
    }
    if (any) cg_flags |= 1ull << g;
  }
  if (!cg_flags) return 0.0;
  const uint16_t *scan = sm_scan(T, scan_idx, log2n - 2);
  const uint8_t *scan_cg = T->scan_cg[scan_idx][log2n - 2];
  int cg_last = ncg - 1;
  while (!((cg_flags >> scan_cg[cg_last]) & 1)) --cg_last;
  int scan_last = cg_last * 16 + 15;
  while (!coeff[scan[scan_last]]) --scan_last;
  const int pos_last = scan[scan_last];

  // every term is an integer multiple of 2^-15 bit: the reference's double sums are exact, so the integer sum (units of
  // 2^-15) converted once gives the same double, without a floating-point add chain per bin
  long long bits = 0;
  if (n == 4 && cfg->trskip_enable) cabac_bin_i(tb, c, type == 0 ? CTX_TRSKIP_LUMA : CTX_TRSKIP_CHROMA, tr_skip, &bits);
  long long bits_last = 0;
  {
    int lx = pos_last & (n - 1), ly = pos_last >> log2n;
    if (scan_idx == 2) { const int t = lx; lx = ly; ly = t; }
    const int idx = log2n - 2;
    const int ctx_offset = type ? 0 : (idx * 3 + (idx + 1) / 4);
    const int shift = type ? idx : (idx + 3) / 4;
    const int base_x = type ? CTX_LAST_X_CHROMA : CTX_LAST_X_LUMA;
    const int base_y = type ? CTX_LAST_Y_CHROMA : CTX_LAST_Y_LUMA;
    const int gx = T->group_idx[lx], gy = T->group_idx[ly], gmax = T->group_idx[n - 1];
    for (int k = 0; k < gx; ++k) cabac_bin_i(tb, c, base_x + ctx_offset + (k >> shift), 1, &bits_last);
    if (gx < gmax) cabac_bin_i(tb, c, base_x + ctx_offset + (gx >> shift), 0, &bits_last);
    for (int k = 0; k < gy; ++k) cabac_bin_i(tb, c, base_y + ctx_offset + (k >> shift), 1, &bits_last);
    if (gy < gmax) cabac_bin_i(tb, c, base_y + ctx_offset + (gy >> shift), 0, &bits_last);
    if (gx > 3) bits_last += (long long)((gx - 2) / 2) << 15;
    if (gy > 3) bits_last += (long long)((gy - 2) / 2) << 15;
  }
  const int base_cg = CTX_SIG_CG + type;
  const int base_sig = type == 0 ? CTX_SIG_LUMA : CTX_SIG_CHROMA;
  int c1 = 1;
  int scan_pos_sig = scan_last;
  for (int i = cg_last; i >= 0; --i) {
    const int sub_pos = i << 4;
    int32_t *abs_coeff = tb->abs_scratch[CTU_HALF & 7];
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
    else cabac_bin_i(tb, c, base_cg + (right || lower), (int)((cg_flags >> cg_blk) & 1), &bits);
    if ((cg_flags >> cg_blk) & 1) {
      const int pattern = (n == 4) ? -1 : right + (lower << 1);
      for (; scan_pos_sig >= sub_pos; --scan_pos_sig) {
        const int blk = scan[scan_pos_sig];
        const int sig = coeff[blk] != 0;
        if (scan_pos_sig > sub_pos || i == 0 || num_nz)
          cabac_bin_i(tb, c, base_sig + sig_ctx_inc(T, pattern, scan_idx, blk & (n - 1), blk >> log2n, log2n, type), sig, &bits);
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
        cabac_bin_i(tb, c, base_one + c1, symbol, &bits);
        if (symbol) { c1 = 0; if (first_c2 == -1) first_c2 = k; }
        else if (c1 < 3 && c1 > 0) ++c1;
      }
      if (c1 == 0 && first_c2 != -1)
        cabac_bin_i(tb, c, (type == 0 ? CTX_ABS_LUMA : CTX_ABS_CHROMA) + ctx_set, abs_coeff[first_c2] > 2, &bits);
      bits += (long long)((cfg->signhide_enable && sign_hidden) ? num_nz - 1 : num_nz) << 15;
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
  return (double)(bits_last + bits) * (1.0 / 32768.0);
}

// ------------------------------------------------------------------------------------------------ one transform unit
// Everything kvz_intra_recon_cu does for one colour of one transform unit (ref: intra.c:561-620 prediction,
// transform.c:294-415 quantize_tr_residual, quant-generic.c:198-292 kvz_quantize_residual), fused and kept in the
// team's scratch: prediction, residual, transform (or transform skip), RDOQ / quantisation, and when a level
// survived dequantisation, inverse transform and reconstruction; plus the SSD against the source that the callers'
// cost functions need (kvz_pixels_calc_ssd).  Results: tu.pred(), tu.q(), tu.rec(), fx->has, fx->ssd.
template <typename Pix> struct TuJob {
  const IntraRefs<Pix> *refs;
  const Pix *src;       // the unit's source pixels
  int src_stride;
  int color, log2n, mode, scan_idx;
  int rdoq_tr_depth;        // context selector of RDOQ's cbf cost (quant-generic.c:237-238)
};

template <int L2N, typename Pix>
CTU_FN_NOINLINE void tu_core_t(const Team &tm, const SmTables *T, const SmTables *tb, const CtuConfig *cfg, const uint8_t *cabac0, const TuS<Pix> &tu,
                               const TuJob<Pix> &j, bool use_trskip)
{
  const int log2n = L2N ? L2N : j.log2n, n = 1 << log2n, nn = n * n;
  const int color = j.color;
  const int ts_shift = 15 - PixDepth<Pix>::bd - log2n;
  int16_t *a = tu.a(), *b = tu.b(), *q = tu.q(), *t = tu.t();
  Pix *pred = tu.pred(), *rec = tu.rec();
  TuFixed<Pix> *fx = tu.fx();
  #pragma unroll 1
  for (int e = tm.tid; e < nn; e += tm.nt) {
    const int y = e >> log2n, x = e & (n - 1);
    const int p = intra_predict_px(j.refs, log2n, j.mode, color, x, y);
    pred[e] = (Pix)p;
    a[e] = (int16_t)((int)j.src[y * j.src_stride + x] - p);
  }
  if (tm.tid == 0) { fx->has = 0; fx->ssd = 0; fx->cg_mask[0] = 0; fx->cg_mask[1] = 0; }
  tsync(tm);
  const bool use_dst = (n == 4 && color == 0);
  const int8_t *M = use_dst ? T->dst4 : sm_tr(T, log2n - 2);
  if (use_trskip) {
    #pragma unroll 1
    for (int e = tm.tid; e < nn; e += tm.nt) b[e] = (int16_t)((uint16_t)a[e] << ts_shift);
    tsync(tm);
  } else {
    fwd_pass<L2N>(tm, a, t, M, n, log2n - 1 + (PixDepth<Pix>::bd - 8));
    fwd_pass<L2N>(tm, t, b, M, n, log2n + 6);
  }
  const int type = color == 0 ? 0 : 2;
  if (cfg->rdoq_enable && (n > 4 || !cfg->rdoq_skip)) {
    const int nl = rdoq_lanes(tm);
    if (tm.tid < nl) rdoq_team<L2N>(T, tb, cfg, cabac0, tu, log2n, type, j.scan_idx, j.rdoq_tr_depth, tm.tid, nl, tm.mask);
    tsync(tm);
  } else {
    quant_block(tm, T, cfg, tu, n, type, j.scan_idx);
  }
  {
    uint32_t m0 = 0, m1 = 0;
    const int side_shift = log2n - 2;
    #pragma unroll 1
    for (int e = tm.tid; e < nn; e += tm.nt) {
      if (q[e] != 0) {
        const int g = (((e >> log2n) >> 2) << side_shift) + ((e & (n - 1)) >> 2);
        if (g < 32) m0 |= 1u << g; else m1 |= 1u << (g - 32);
      }
    }
    if (m0) CTU_ATOMIC_OR(&fx->cg_mask[0], m0);
    if (m1) CTU_ATOMIC_OR(&fx->cg_mask[1], m1);
    if (m0 | m1) CTU_ATOMIC_OR(&fx->has, 1);
  }
  tsync(tm);
  int ssd = 0;
  if (fx->has) {
    dequant_block<L2N>(tm, cfg, tu, n, color == 0 ? 0 : (color == 1 ? 2 : 3));
    if (use_trskip) {
      const int offs = 1 << (ts_shift - 1);
      #pragma unroll 1
      for (int e = tm.tid; e < nn; e += tm.nt) a[e] = (int16_t)(((int)b[e] + offs) >> ts_shift);
      tsync(tm);
    } else {
      inv_pass<L2N>(tm, b, t, M, n, 7);
      inv_pass<L2N>(tm, t, a, M, n, 12 - (PixDepth<Pix>::bd - 8));
    }
    #pragma unroll 1
    for (int e = tm.tid; e < nn; e += tm.nt) {
      const int y = e >> log2n, x = e & (n - 1);
      const int16_t val = (int16_t)(a[e] + (int)pred[e]);
      const int r = iclip(0, PixTraits<Pix>::max, (int)val);
      rec[e] = (Pix)r;
      const int d = (int)j.src[y * j.src_stride + x] - r;
      ssd += d * d;
    }
  } else {
    #pragma unroll 1
    for (int e = tm.tid; e < nn; e += tm.nt) {
      const int y = e >> log2n, x = e & (n - 1);
      const int r = pred[e];
      rec[e] = (Pix)r;
      const int d = (int)j.src[y * j.src_stride + x] - r;
      ssd += d * d;
    }
  }
  if (ssd) CTU_ATOMIC_ADD(&fx->ssd, ssd);
  tsync(tm);
  if constexpr (PixDepth<Pix>::bd != 8) {
    // kvz_pixels_calc_ssd scales the unit's SSD to 8-bit precision (picture-generic.c:550)
    if (tm.tid == 0) fx->ssd >>= 2 * (PixDepth<Pix>::bd - 8);
    tsync(tm);
  }
}

template <typename Pix> CTU_FN void tu_core(const Team &tm, const SmTables *T, const SmTables *tb, const CtuConfig *cfg, const uint8_t *cabac0, const TuS<Pix> &tu,
                    const TuJob<Pix> &j, bool use_trskip)
{
  if (j.log2n == 2) tu_core_t<2>(tm, T, tb, cfg, cabac0, tu, j, use_trskip);
  else tu_core_t<0>(tm, T, tb, cfg, cabac0, tu, j, use_trskip);
}

// One colour of one transform unit including the transform-skip decision of 4x4 luma units
// (kvz_quantize_residual_trskip, ref: transform.c:242-288).  `sc`: the search models the decision's bit costs read.
// Returns tr_skip (uniform over the team); the chosen alternative is in tu.q() / tu.rec() / fx->has / fx->ssd.
template <typename Pix> CTU_FN_NOINLINE int tu_eval(const Team &tm, const SmTables *T, const SmTables *tb, const CtuConfig *cfg, const uint8_t *cabac0, CabacState *sc,
                            const TuS<Pix> &tu, const TuJob<Pix> &j)
{
  if (!(j.log2n == 2 && j.color == 0 && cfg->trskip_enable)) {
    tu_core(tm, T, tb, cfg, cabac0, tu, j, false);
    return 0;
  }
  TuFixed<Pix> *fx = tu.fx();
  for (int k = 0; k < 2; ++k) {
    tu_core(tm, T, tb, cfg, cabac0, tu, j, k == 1);
    #pragma unroll 1
    for (int e = tm.tid; e < 16; e += tm.nt) { fx->ts_rec[k][e] = tu.rec()[e]; fx->ts_coeff[k][e] = tu.q()[e]; }
    if (tm.tid == 0) { fx->ts_has[k] = fx->has; fx->ts_ssd[k] = fx->ssd; fx->ts_mask[k] = fx->cg_mask[0]; }
    tsync(tm);
  }
  if (tm.tid == 0) {
    double cost[2];
    for (int k = 0; k < 2; ++k) {
      cost[k] = (double)(unsigned)fx->ts_ssd[k];
      cost[k] += coeff_cost_serial(T, tb, cfg, sc, fx->ts_coeff[k], 2, 0, j.scan_idx, 0, fx->ts_mask[k]) * cfg->lambda;
    }
    fx->ts_pick = cost[0] <= cost[1] ? 0 : 1;
  }
  tsync(tm);
  const int pick = fx->ts_pick;
  // (the second alternative is still in place when it wins)
  if (pick == 0) {
    #pragma unroll 1
    for (int e = tm.tid; e < 16; e += tm.nt) { tu.q()[e] = fx->ts_coeff[0][e]; tu.rec()[e] = fx->ts_rec[0][e]; }
    if (tm.tid == 0) { fx->has = fx->ts_has[0]; fx->ssd = fx->ts_ssd[0]; fx->cg_mask[0] = fx->ts_mask[0]; fx->cg_mask[1] = 0; }
    tsync(tm);
  }
  return pick;
}

}  // namespace kvzctu
