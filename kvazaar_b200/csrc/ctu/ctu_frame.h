// ctu_frame.h -- what surrounds the search of a CTU inside the CTU job (ref: encoder_state_worker_encode_lcu,
// src/encoderstate.c:636-773): loading the CTU's neighbourhood (init_lcu_t, search.c:1076-1170), storing its
// decisions (copy_lcu_to_cu_data :1176-1201, encoder_state_recdata_to_bufs encoderstate.c:192-253), deblocking
// (kvz_filter_deblock_lcu, filter.c:783-792), the SAO parameter search (kvz_sao_search_lcu, sao.c:671-735) and the
// adaptation of the REAL coder's context models by the CTU's syntax (encode_sao encoderstate.c:467-552,
// kvz_encode_coding_tree encode_coding_tree.c:745-975) -- the next CTU's search starts from those models
// (search.c:1211), so they are tracked on the device; the bits themselves are written by the host.
#pragma once
#include "ctu_search.h"

namespace kvzctu {

// Device-resident state of one frame in flight.
template <typename Pix> struct FrameDevT {
  const Pix *src_y, *src_u, *src_v;     // source planes, stride = width (/2)
  Pix *rec_y, *rec_u, *rec_v;           // reconstruction: search output, then deblocked in place
  Pix *out_y, *out_u, *out_v;           // final picture (after SAO)
  Pix *dbg_y, *dbg_u, *dbg_v;           // optional: the search's reconstruction before deblocking (verification)
  Pix *hor_y, *hor_u, *hor_v;           // hor_buf_search: un-deblocked bottom row of every CTU row
  Pix *ver_y, *ver_u, *ver_v;           // ver_buf_search: un-deblocked right column of every CTU column
  CuRec *cu;                                // per 4x4, stride cu_stride
  int16_t *coeff;                           // per CTU: y[4096] u[1024] v[1024]
  SaoRec *sao;                              // per CTU: [2] luma, chroma
  CabacState *row_ctx;                      // per CTU row: the real coder's models (state->cabac) of that row
  int32_t cu_stride;
  int32_t wlcu, hlcu;
};
using FrameDev = FrameDevT<uint8_t>;  // (8-bit alias, see CtuWork)

// ------------------------------------------------------------------------------------------------ init_lcu_t
template <typename Pix> CTU_FN_NOINLINE void ctu_load(CtuST<Pix> *S, const FrameDevT<Pix> *F, int cx, int cy)
{
  S = sm(S);
  const CtuConfig *cfg = &S->cfg;
  CtuWorkT<Pix> *W = S->W;
  LcuLevel<Pix> *L0 = &S->lv[0];
  const int x = cx * 64, y = cy * 64;
  const int Wd = cfg->width, H = cfg->height;
  // FILL(*lcu, 0) for every level of the work tree (work_tree[depth] = work_tree[0] below only differs in the border
  // CU records), and the levels' plane pointers
  {
    #pragma unroll 1
    for (int d = CTU_TID; d < 5; d += CTU_NT) {
      LcuLevel<Pix> *L = &S->lv[d];
      LcuStore<Pix> *st = &W->store[d];
      L->rec_y = st->rec_y; L->rec_u = st->rec_u; L->rec_v = st->rec_v;
      L->coeff_y = st->coeff_y; L->coeff_u = st->coeff_u; L->coeff_v = st->coeff_v;
    }
    uint32_t *p = (uint32_t *)W->store;
    #pragma unroll 1
    for (int i = CTU_TID; i < (int)(5 * sizeof(LcuStore<Pix>) / 4); i += CTU_NT) p[i] = 0;
    uint32_t *q = (uint32_t *)L0->cu;
    #pragma unroll 1
    for (int i = CTU_TID; i < (int)(sizeof(L0->cu) / 4); i += CTU_NT) q[i] = 0;
    #pragma unroll 1
    for (int i = CTU_TID; i < 4096; i += CTU_NT) W->src_y[i] = 0;
    #pragma unroll 1
    for (int i = CTU_TID; i < 1024; i += CTU_NT) { W->src_u[i] = 0; W->src_v[i] = 0; }
    #pragma unroll 1
    for (int i = CTU_TID; i < 100; i += CTU_NT) { W->top_y[i] = 0; W->left_y[i] = 0; }
    #pragma unroll 1
    for (int i = CTU_TID; i < 52; i += CTU_NT) { W->top_u[i] = 0; W->top_v[i] = 0; W->left_u[i] = 0; W->left_v[i] = 0; }
  }
  CTU_SYNC();
  // neighbouring CU records
  #pragma unroll 1
  for (int i = CTU_TID; i < 16; i += CTU_NT) {
    if (y > 0 && x + 4 * i < Wd) *cu_at(L0, 4 * i, -1) = ld_frame_cu(&F->cu[((y - 1) >> 2) * F->cu_stride + ((x + 4 * i) >> 2)]);
    if (x > 0 && y + 4 * i < H) *cu_at(L0, -1, 4 * i) = ld_frame_cu(&F->cu[((y + 4 * i) >> 2) * F->cu_stride + ((x - 1) >> 2)]);
  }
  CTU_LEADER {
    if (x > 0 && y > 0) *cu_at(L0, -1, -1) = ld_frame_cu(&F->cu[((y - 1) >> 2) * F->cu_stride + ((x - 1) >> 2)]);
    if (y > 0 && x + 64 < Wd) *cu_top_right(L0) = ld_frame_cu(&F->cu[((y - 1) >> 2) * F->cu_stride + ((x + 64) >> 2)]);
  }
  // reference pixels: index 0 of the border arrays is the top-left corner sample
  if (y > 0) {
    const int x_max = imin(96, Wd - x);
    const int x_min = x > 0 ? 0 : 1;
    // luma: entries x_min .. x_max (entry e = picture column x + e - 1) from the bottom row of CTU row cy - 1
    #pragma unroll 1
    for (int e = x_min + CTU_TID; e <= x_max; e += CTU_NT) W->top_y[e] = CTU_LD_FRAME(&F->hor_y[(cy - 1) * Wd + x + e - 1]);
    #pragma unroll 1
    for (int e = x_min + CTU_TID; e <= x_max / 2; e += CTU_NT) {
      W->top_u[e] = CTU_LD_FRAME(&F->hor_u[(cy - 1) * (Wd / 2) + x / 2 + e - 1]);
      W->top_v[e] = CTU_LD_FRAME(&F->hor_v[(cy - 1) * (Wd / 2) + x / 2 + e - 1]);
    }
  }
  if (x > 0) {
    const int y_min = y > 0 ? 0 : 1;
    // entries y_min .. 64 from the right column of CTU column cx - 1; rows below the picture are not copied by
    // the reference either way of interest (they are never read: availability is clipped to the picture)
    #pragma unroll 1
    for (int e = y_min + CTU_TID; e <= 64; e += CTU_NT) { const int yy = y + e - 1; if (yy < H) W->left_y[e] = CTU_LD_FRAME(&F->ver_y[(cx - 1) * H + yy]); }
    #pragma unroll 1
    for (int e = y_min + CTU_TID; e <= 32; e += CTU_NT) {
      const int yy = y / 2 + e - 1;
      if (yy < H / 2) { W->left_u[e] = CTU_LD_FRAME(&F->ver_u[(cx - 1) * (H / 2) + yy]); W->left_v[e] = CTU_LD_FRAME(&F->ver_v[(cx - 1) * (H / 2) + yy]); }
    }
  }
  // source pixels
  {
    const int x_max = imin(x + 64, Wd) - x, y_max = imin(y + 64, H) - y;
    #pragma unroll 1
    for (int e = CTU_TID; e < 64 * 64; e += CTU_NT) { const int yy = e >> 6, xx = e & 63; if (xx < x_max && yy < y_max) W->src_y[e] = F->src_y[(y + yy) * Wd + x + xx]; }
    #pragma unroll 1
    for (int e = CTU_TID; e < 32 * 32; e += CTU_NT) {
      const int yy = e >> 5, xx = e & 31;
      if (xx < x_max / 2 && yy < y_max / 2) {
        W->src_u[e] = F->src_u[(y / 2 + yy) * (Wd / 2) + x / 2 + xx];
        W->src_v[e] = F->src_v[(y / 2 + yy) * (Wd / 2) + x / 2 + xx];
      }
    }
  }
  CTU_SYNC();
  // work_tree[depth] = work_tree[0]
  for (int d = 1; d <= 4; ++d) {
    const uint32_t *s = (const uint32_t *)L0->cu;
    uint32_t *p = (uint32_t *)S->lv[d].cu;
    #pragma unroll 1
    for (int i = CTU_TID; i < (int)(sizeof(L0->cu) / 4); i += CTU_NT) p[i] = s[i];
  }
  // the models the search starts from
  #pragma unroll 1
  for (int i = CTU_TID; i < (int)(sizeof(CabacState) / 4); i += CTU_NT) ((uint32_t *)&S->cabac0)[i] = CTU_LD_FRAME((const uint32_t *)&F->row_ctx[cy] + i);
  CTU_SYNC();
  CTU_LEADER { S->cabac0.update = 0; S->sc = S->cabac0; }
  CTU_SYNC();
}

// ------------------------------------------------------------------------------------------------ store
template <typename Pix> CTU_FN_NOINLINE void ctu_store(CtuST<Pix> *S, const FrameDevT<Pix> *F, int cx, int cy)
{
  S = sm(S);
  const CtuConfig *cfg = &S->cfg;
  LcuLevel<Pix> *L0 = &S->lv[0];
  const int x = cx * 64, y = cy * 64, Wd = cfg->width, H = cfg->height;
  const int x_max = imin(x + 64, Wd) - x, y_max = imin(y + 64, H) - y;
  #pragma unroll 1
  for (int e = CTU_TID; e < 256; e += CTU_NT) {
    const int sx = e & 15, sy = e >> 4;
    if (4 * sx < x_max && 4 * sy < y_max) F->cu[((y >> 2) + sy) * F->cu_stride + (x >> 2) + sx] = *cu_at(L0, 4 * sx, 4 * sy);
  }
  #pragma unroll 1
  for (int e = CTU_TID; e < 64 * 64; e += CTU_NT) {
    const int yy = e >> 6, xx = e & 63;
    if (xx < x_max && yy < y_max) {
      const Pix v = L0->rec_y[e];
      F->rec_y[(y + yy) * Wd + x + xx] = v;
      if (F->dbg_y) F->dbg_y[(y + yy) * Wd + x + xx] = v;
      if (yy == y_max - 1) F->hor_y[cy * Wd + x + xx] = v;
      if (xx == x_max - 1) F->ver_y[cx * H + y + yy] = v;
    }
  }
  #pragma unroll 1
  for (int e = CTU_TID; e < 32 * 32; e += CTU_NT) {
    const int yy = e >> 5, xx = e & 31;
    if (xx < x_max / 2 && yy < y_max / 2) {
      const Pix u = L0->rec_u[e], v = L0->rec_v[e];
      const int o = (y / 2 + yy) * (Wd / 2) + x / 2 + xx;
      F->rec_u[o] = u; F->rec_v[o] = v;
      if (F->dbg_u) { F->dbg_u[o] = u; F->dbg_v[o] = v; }
      if (yy == y_max / 2 - 1) { F->hor_u[cy * (Wd / 2) + x / 2 + xx] = u; F->hor_v[cy * (Wd / 2) + x / 2 + xx] = v; }
      if (xx == x_max / 2 - 1) { F->ver_u[cx * (H / 2) + y / 2 + yy] = u; F->ver_v[cx * (H / 2) + y / 2 + yy] = v; }
    }
  }
  int16_t *co = F->coeff + (size_t)(cy * F->wlcu + cx) * 6144;
  #pragma unroll 1
  for (int e = CTU_TID; e < 4096; e += CTU_NT) co[e] = L0->coeff_y[e];
  #pragma unroll 1
  for (int e = CTU_TID; e < 1024; e += CTU_NT) { co[4096 + e] = L0->coeff_u[e]; co[5120 + e] = L0->coeff_v[e]; }
  CTU_SYNC();
}

// ------------------------------------------------------------------------------------------------ deblocking
CTU_FN int dbk_tc(int i)
{
  const uint8_t t[54] = { PIX_DBK_TC };
  return t[i];
}
template <typename Pix> CTU_FN const CuRec *fcu(const FrameDevT<Pix> *F, int x, int y) { return &F->cu[(y >> 2) * F->cu_stride + (x >> 2)]; }

// is the left (top) edge of the 8x8 unit at (x, y) a TU or PU boundary (ref: filter.c:194-246)
template <typename Pix> CTU_FN bool dbk_edge_wanted(const FrameDevT<Pix> *F, int x, int y, bool hor)
{
  const CuRec s = ld_frame_cu(fcu(F, x, y));
  const int tu_w = 64 >> s.tr_depth, cu_w = 64 >> s.depth;
  const int pos = hor ? y : x;
  if ((pos & (tu_w - 1)) == 0) return true;
  const int cu_pos = pos & ~(cu_w - 1);
  return pos == cu_pos;       // (the inner PU boundary of NxN lies off the 8x8 grid)
}

// the deblocking filters (dbk_luma_part, dbk_chroma_part: pixel_rules.h) on the frame planes, read through L2; the luma
// filter is a call of its own
struct FrameLoad { template <typename Pix> CTU_MFN int operator()(const Pix *p) const { return CTU_LD_FRAME(p); } };
template <typename Pix> CTU_FN_NOINLINE void dbk_luma_frame(Pix *px, int xs, int ys, int beta, int tc) { dbk_luma_part<Pix>(px, xs, ys, beta, tc, FrameLoad()); }
template <typename Pix> CTU_FN void dbk_chroma_frame(Pix *px, int xs, int ys, int tc) { dbk_chroma_part<Pix>(px, xs, ys, tc, FrameLoad()); }

// kvz_filter_deblock_lcu on the frame planes; all CUs are intra (boundary strength 2), fixed QP
template <typename Pix> CTU_FN_NOINLINE void ctu_deblock(CtuST<Pix> *S, const FrameDevT<Pix> *F, int cx, int cy)
{
  S = sm(S);
  const CtuConfig *cfg = &S->cfg;
  const int Wd = cfg->width, H = cfg->height, Wc = Wd / 2;
  const int x0 = cx * 64, y0 = cy * 64;
  const int end_x = imin(x0 + 64, Wd), end_y = imin(y0 + 64, H);
  const int qp = cfg->qp;
  const int scale = 1 << (PixTraits<Pix>::bd - 8);          // bitdepth_scale (ref: filter.c:373, 590)
  const int beta = dbk_beta(iclip(0, 51, qp + 2 * cfg->deblock_beta)) * scale;
  const int tc_l = dbk_tc(iclip(0, 53, qp + 2 + 2 * cfg->deblock_tc)) * scale;
  const int tc_c = dbk_tc(iclip(0, 53, scaled_qp(2, qp, 0) + 2 + 2 * cfg->deblock_tc)) * scale;
  const int ux_n = (end_x - x0) / 8, uy_n = (end_y - y0) / 8;
  // pass 1: vertical edges of every 8x8 unit: two luma parts per unit, one chroma part where x % 16 == 0
  #pragma unroll 1
  for (int it = CTU_TID; it < ux_n * uy_n * 3; it += CTU_NT) {
    const int part = it % 3, u = it / 3;
    const int ex = x0 + (u % ux_n) * 8, ey = y0 + (u / ux_n) * 8;
    if (ex == 0) continue;
    if (!dbk_edge_wanted(F, ex, ey, false)) continue;
    if (part < 2) dbk_luma_frame(F->rec_y + (size_t)(ey + 4 * part) * Wd + ex, 1, Wd, beta, tc_l);
    else if ((ex & 15) == 0) {
      dbk_chroma_frame(F->rec_u + (size_t)(ey / 2) * Wc + ex / 2, 1, Wc, tc_c);
      dbk_chroma_frame(F->rec_v + (size_t)(ey / 2) * Wc + ex / 2, 1, Wc, tc_c);
    }
  }
  CTU_SYNC();
#if defined(__CUDA_ARCH__)
  __threadfence();
#endif
  // pass 2: horizontal edges: the delayed rightmost four columns of the CTU to the left, then this CTU's units
  // (without their own rightmost four columns unless the CTU ends the picture row)
  const int left_items = x0 > 0 ? uy_n : 0;
  #pragma unroll 1
  for (int it = CTU_TID; it < left_items + ux_n * uy_n * 3; it += CTU_NT) {
    if (it < left_items) {
      const int ey = y0 + it * 8, ex = x0 - 8;          // unit holding the delayed columns
      if (ey == 0) continue;
      if (!dbk_edge_wanted(F, x0 - 4, ey, true)) continue;
      dbk_luma_frame(F->rec_y + (size_t)ey * Wd + x0 - 4, Wd, 1, beta, tc_l);
      if ((ey & 15) == 0) {
        dbk_chroma_frame(F->rec_u + (size_t)(ey / 2) * Wc + x0 / 2 - 4, Wc, 1, tc_c);
        dbk_chroma_frame(F->rec_v + (size_t)(ey / 2) * Wc + x0 / 2 - 4, Wc, 1, tc_c);
      }
      (void)ex;
      continue;
    }
    const int j = it - left_items;
    const int part = j % 3, u = j / 3;
    const int ex = x0 + (u % ux_n) * 8, ey = y0 + (u / ux_n) * 8;
    if (ey == 0) continue;
    if (!dbk_edge_wanted(F, ex, ey, true)) continue;
    const bool delayed = ((ex + 8) % 64 == 0) && (ex + 8 != Wd);
    if (part == 0) dbk_luma_frame(F->rec_y + (size_t)ey * Wd + ex, Wd, 1, beta, tc_l);
    else if (part == 1) { if (!delayed) dbk_luma_frame(F->rec_y + (size_t)ey * Wd + ex + 4, Wd, 1, beta, tc_l); }
    else if ((ey & 15) == 0 && !delayed) {
      dbk_chroma_frame(F->rec_u + (size_t)(ey / 2) * Wc + ex / 2, Wc, 1, tc_c);
      dbk_chroma_frame(F->rec_v + (size_t)(ey / 2) * Wc + ex / 2, Wc, 1, tc_c);
    }
  }
  CTU_SYNC();
}

// ------------------------------------------------------------------------------------------------ SAO search
struct SaoStats {
  int32_t edge[3][4][2][5];     // [plane][class][sum, count][category]
  int32_t band[3][2][32];       // [plane][sum, count][band]
};

// statistics of the CTU's block of one plane (the reference works on a contiguous copy: same pixels)
template <typename Pix> CTU_FN_NOINLINE void sao_stats_plane(const Pix *org, const Pix *rec, int stride, int bw, int bh, int32_t edge[4][2][5], int32_t band[2][32])
{
  // bands: the top five bits of the sample (ref: sao.c:273); edge sums: differences rounded to 8-bit precision
  // (ref: sao-generic.c:66-77)
  constexpr int band_shift = PixTraits<Pix>::bd - 5, edge_shift = PixTraits<Pix>::bd - 8;
  constexpr int edge_round = edge_shift ? 1 << (edge_shift - 1) : 0;
  #pragma unroll 1
  for (int e = CTU_TID; e < bw * bh; e += CTU_NT) {
    const int y = e / bw, x = e - y * bw;
    const int cc = CTU_LD_FRAME(&rec[y * stride + x]), d = (int)org[y * stride + x] - cc;
    CTU_ATOMIC_ADD(&band[0][cc >> band_shift], d);
    CTU_ATOMIC_ADD(&band[1][cc >> band_shift], 1);
    if (x >= 1 && x < bw - 1 && y >= 1 && y < bh - 1) {
      for (int k = 0; k < 4; ++k) {
        int ax, ay;
        sao_eo_offsets(k, ax, ay);
        const int a = CTU_LD_FRAME(&rec[(y + ay) * stride + x + ax]), b = CTU_LD_FRAME(&rec[(y - ay) * stride + x - ax]);
        const int cat = sao_eo_cat(a, b, cc);
        CTU_ATOMIC_ADD(&edge[k][0][cat], (d + edge_round) >> edge_shift);
        CTU_ATOMIC_ADD(&edge[k][1][cat], 1);
      }
    }
  }
}

// the leader-only part: sao.c:55-160 (mode bits), 208-258 (band offsets), 364-603 (best mode + merge costs)
struct SaoBits { const SmTables *T; const uint8_t *ctx; };
CTU_FN double sao_fbits(const SaoBits &b, int off, int val) { return (double)b.T->ebits[b.ctx[off] ^ val] * (1.0 / 32768.0); }
CTU_FN double sao_bits_prefix(const SaoBits &b, bool has_left, bool has_top, int type_bin)
{
  double m = 0.0;
  if (has_left) m += sao_fbits(b, CTX_SAO_MERGE, 0);
  if (has_top) m += sao_fbits(b, CTX_SAO_MERGE, 0);
  m += sao_fbits(b, CTX_SAO_TYPE, type_bin);
  return m;
}
template <typename Pix> CTU_FN double sao_mode_bits_edge(const SaoBits &b, const int *offsets, bool has_top, bool has_left, int buf_cnt)
{
  double m = sao_bits_prefix(b, has_left, has_top, 1);
  m += 1.0;
  for (int bi = 0; bi < buf_cnt; ++bi)
    for (int cat = 1; cat <= 4; ++cat) {
      const int a = iabs(offsets[cat + 5 * bi]);
      if (a == 0 || a == PixTraits<Pix>::sao_max) m += a + 1; else m += a + 2;
    }
  m += 2.0;
  return m;
}
template <typename Pix> CTU_FN double sao_mode_bits_band(const SaoBits &b, const int *offsets, bool has_top, bool has_left, int buf_cnt)
{
  double m = sao_bits_prefix(b, has_left, has_top, 1);
  m += 1.0;
  for (int bi = 0; bi < buf_cnt; ++bi)
    for (int i = 0; i < 4; ++i) {
      const int a = iabs(offsets[i + 1 + bi * 5]);
      if (a == 0) m += a + 1; else if (a == PixTraits<Pix>::sao_max) m += a + 1 + 1; else m += a + 2 + 1;
    }
  m += 5.0 * buf_cnt;
  return m;
}
CTU_FN int sao_edge_ddist(const int32_t st[2][5], const int *offsets /* [5] */)
{
  int sum = 0;
  for (int cat = 0; cat < 5; ++cat) { const int o = offsets[cat]; if (o != 0) sum += st[1][cat] * o * o - 2 * o * st[0][cat]; }
  return sum;
}
CTU_FN int sao_band_ddist(const int32_t bd[2][32], int band_pos, const int *offs /* [4] */)
{
  int sum = 0;
  for (int k = 0; k < 4; ++k) { const int o = offs[k], bi = band_pos + k; if (o != 0 && bi >= 0 && bi < 32) sum += bd[1][bi] * o * o - 2 * o * bd[0][bi]; }
  return sum;
}
template <typename Pix> CTU_FN_NOINLINE int sao_band_offsets(const int32_t bd[2][32], int *offsets /* [4] */, int *band_position)
{
  int dist[32], temp_offsets[32];
  for (int band = 0; band < 32; ++band) {
    int best_dist = CTU_MAX_INT, offset = 0;
    if (bd[1][band] != 0) { offset = (bd[0][band] + (bd[1][band] >> 1)) / bd[1][band]; offset = iclip(-PixTraits<Pix>::sao_max, PixTraits<Pix>::sao_max, offset); }
    dist[band] = offset == 0 ? 0 : CTU_MAX_INT;
    temp_offsets[band] = 0;
    while (offset != 0) {
      const int temp_dist = bd[1][band] * offset * offset - 2 * offset * bd[0][band];
      if (temp_dist < best_dist) { dist[band] = temp_dist; temp_offsets[band] = offset; }   // (best_dist is never lowered: the reference's quirk)
      offset += (offset > 0) ? -1 : 1;
    }
  }
  int best_dist = CTU_MAX_INT, best_pos = 0;
  for (int band = 0; band < 28; ++band) {
    // the reference adds four ints that may each be INT_MAX: unsigned wrap-around reproduces the signed overflow of x86
    const int temp_dist = (int)((unsigned)dist[band] + (unsigned)dist[band + 1] + (unsigned)dist[band + 2] + (unsigned)dist[band + 3]);
    if (temp_dist < best_dist) { best_dist = temp_dist; best_pos = band; }
  }
  for (int k = 0; k < 4; ++k) offsets[k] = temp_offsets[best_pos + k];
  *band_position = best_pos;
  return best_dist;
}

// sao_search_best_mode for one component group (luma: planes {0}, chroma: planes {1, 2}).  Leader only.
template <typename Pix> CTU_FN_NOINLINE void sao_search_best_mode(CtuST<Pix> *S, const SaoStats *st, int first_plane, int buf_cnt, SaoRec *out, const SaoRec *top, const SaoRec *left, int32_t merge_cost[3])
{
  S = sm(S); st = sm(st);
  const CtuConfig *cfg = &S->cfg;
  const SaoBits sb = { &S->tb, S->cabac0.ctx };
  const double lambda = cfg->lambda;
  SaoRec edge, band;
  memset(&edge, 0, sizeof(edge)); memset(&band, 0, sizeof(band));
  if (cfg->sao_type & 1) {
    edge.type = 2; edge.ddistortion = CTU_MAX_INT;
    for (int cls = 0; cls < 4; ++cls) {
      int eo[10];
      for (int i = 0; i < 10; ++i) eo[i] = 0;
      int sum_dd = 0;
      for (int i = 0; i < buf_cnt; ++i) {
        const int32_t (*s)[5] = st->edge[first_plane + i][cls];
        for (int cat = 1; cat <= 4; ++cat) {
          const int cat_sum = s[0][cat], cat_cnt = s[1][cat];
          int offset = 0;
          if (cat_cnt != 0) { offset = (cat_sum + (cat_cnt >> 1)) / cat_cnt; offset = iclip(-PixTraits<Pix>::sao_max, PixTraits<Pix>::sao_max, offset); }
          if (cat <= 2 && offset < 0) offset = 0;
          if (cat >= 3 && offset > 0) offset = 0;
          eo[cat + 5 * i] = offset;
          sum_dd += cat_cnt * offset * offset - 2 * offset * cat_sum;
        }
      }
      {
        const float mode_bits = (float)sao_mode_bits_edge<Pix>(sb, eo, top != NULL, left != NULL, buf_cnt);
        sum_dd += (int)((double)mode_bits * lambda + 0.5);
      }
      eo[0] = 0; eo[5] = 0;
      if (sum_dd < edge.ddistortion) { edge.eo_class = cls; edge.ddistortion = sum_dd; for (int i = 0; i < 10; ++i) edge.offsets[i] = eo[i]; }
    }
    const float mode_bits = (float)sao_mode_bits_edge<Pix>(sb, edge.offsets, top != NULL, left != NULL, buf_cnt);
    int dd = (int)(mode_bits * lambda + 0.5);
    for (int i = 0; i < buf_cnt; ++i) dd += sao_edge_ddist(st->edge[first_plane + i][edge.eo_class], &edge.offsets[5 * i]);
    edge.ddistortion = dd;
  } else edge.ddistortion = CTU_MAX_INT;
  if (cfg->sao_type & 2) {
    band.type = 1; band.ddistortion = CTU_MAX_INT;
    int temp_offsets[10];
    for (int i = 0; i < 10; ++i) temp_offsets[i] = 0;
    int dd = 0;
    for (int i = 0; i < buf_cnt; ++i) dd += sao_band_offsets<Pix>(st->band[first_plane + i], &temp_offsets[1 + 5 * i], &band.band_position[i]);
    const float temp_rate = (float)sao_mode_bits_band<Pix>(sb, temp_offsets, top != NULL, left != NULL, buf_cnt);
    dd += (int)((double)temp_rate * lambda + 0.5);
    if (dd < band.ddistortion) { band.ddistortion = dd; for (int i = 0; i < buf_cnt * 5; ++i) band.offsets[i] = temp_offsets[i]; }
    const float mode_bits = (float)sao_mode_bits_band<Pix>(sb, band.offsets, top != NULL, left != NULL, buf_cnt);
    int d2 = (int)(mode_bits * lambda + 0.5);
    for (int i = 0; i < buf_cnt; ++i) d2 += sao_band_ddist(st->band[first_plane + i], band.band_position[i], &band.offsets[1 + 5 * i]);
    band.ddistortion = d2;
  } else band.ddistortion = CTU_MAX_INT;
  if (edge.ddistortion <= band.ddistortion) { *out = edge; merge_cost[0] = edge.ddistortion; }
  else { *out = band; merge_cost[0] = band.ddistortion; }
  {
    const float none_bits = (float)sao_bits_prefix(sb, left != NULL, top != NULL, 0);
    const int cost_of_nothing = (int)(none_bits * lambda + 0.5);
    if (out->ddistortion >= cost_of_nothing) { out->type = 0; merge_cost[0] = cost_of_nothing; }
  }
  const SaoRec *cand[2] = { left, top };
  for (int i = 0; i < 2; ++i) {
    const SaoRec *m = cand[i];
    if (!m) continue;
    double mb = 0.0;
    mb += sao_fbits(sb, CTX_SAO_MERGE, i + 1 == 1);
    if (i + 1 != 1) mb += sao_fbits(sb, CTX_SAO_MERGE, i + 1 == 2);
    const float mode_bits = (float)mb;
    int dd = (int)(mode_bits * lambda + 0.5);
    if (m->type == 2) { for (int b = 0; b < buf_cnt; ++b) dd += sao_edge_ddist(st->edge[first_plane + b][m->eo_class], &m->offsets[5 * b]); }
    else if (m->type == 1) { for (int b = 0; b < buf_cnt; ++b) dd += sao_band_ddist(st->band[first_plane + b], m->band_position[b], &m->offsets[1 + 5 * b]); }
    merge_cost[i + 1] = dd;
  }
}

// kvz_sao_search_lcu; `st` is scratch for the statistics in shared memory (the arena, idle after the search)
template <typename Pix> CTU_FN_NOINLINE void ctu_sao_search(CtuST<Pix> *S, const FrameDevT<Pix> *F, SaoStats *st, int cx, int cy)
{
  S = sm(S); st = sm(st);
  const CtuConfig *cfg = &S->cfg;
  const int Wd = cfg->width, H = cfg->height;
  const int x0 = cx * 64, y0 = cy * 64;
  const int bw = imin(64, Wd - x0), bh = imin(64, H - y0);
  {
    int32_t *p = (int32_t *)st;
    #pragma unroll 1
    for (int i = CTU_TID; i < (int)(sizeof(SaoStats) / 4); i += CTU_NT) p[i] = 0;
  }
  CTU_SYNC();
#if defined(__CUDA_ARCH__)
  __threadfence();
#endif
  sao_stats_plane(F->src_y + (size_t)y0 * Wd + x0, F->rec_y + (size_t)y0 * Wd + x0, Wd, bw, bh, st->edge[0], st->band[0]);
  sao_stats_plane(F->src_u + (size_t)(y0 / 2) * (Wd / 2) + x0 / 2, F->rec_u + (size_t)(y0 / 2) * (Wd / 2) + x0 / 2, Wd / 2, bw / 2, bh / 2, st->edge[1], st->band[1]);
  sao_stats_plane(F->src_v + (size_t)(y0 / 2) * (Wd / 2) + x0 / 2, F->rec_v + (size_t)(y0 / 2) * (Wd / 2) + x0 / 2, Wd / 2, bw / 2, bh / 2, st->edge[2], st->band[2]);
  CTU_SYNC();
  CTU_LEADER {
    SaoRec *sl = &F->sao[2 * (cy * F->wlcu + cx)], *sc = sl + 1;
    // the neighbours' parameters were written by other CTAs: local copies through L2
    SaoRec nb[4];      // top luma, top chroma, left luma, left chroma
    if (cy) { const int32_t *q = (const int32_t *)&F->sao[2 * ((cy - 1) * F->wlcu + cx)]; for (int i = 0; i < (int)(2 * sizeof(SaoRec) / 4); ++i) ((int32_t *)&nb[0])[i] = CTU_LD_FRAME(q + i); }
    if (cx) { const int32_t *q = (const int32_t *)&F->sao[2 * (cy * F->wlcu + cx - 1)]; for (int i = 0; i < (int)(2 * sizeof(SaoRec) / 4); ++i) ((int32_t *)&nb[2])[i] = CTU_LD_FRAME(q + i); }
    const SaoRec *top_l = cy ? &nb[0] : NULL, *left_l = cx ? &nb[2] : NULL;
    const SaoRec *top_c = top_l ? top_l + 1 : NULL, *left_c = left_l ? left_l + 1 : NULL;
    int32_t mcl[3] = { CTU_MAX_INT, 0, 0 }, mcc[3] = { CTU_MAX_INT, 0, 0 };
    sao_search_best_mode(S, st, 0, 1, sl, top_l, left_l, mcl);
    sao_search_best_mode(S, st, 1, 2, sc, top_c, left_c, mcc);
    sl->merge_up_flag = sl->merge_left_flag = 0;
    if (top_l) {
      if (mcl[2] + mcc[2] <= mcl[0] + mcc[0]) { *sl = *top_l; *sc = *top_c; sl->merge_up_flag = 1; sl->merge_left_flag = 0; }
    }
    if (left_l) {
      if (mcl[1] + mcc[1] <= mcl[0] + mcc[0]) {
        if (!sl->merge_up_flag || mcl[1] + mcc[1] < mcl[2] + mcc[2]) { *sl = *left_l; *sc = *left_c; sl->merge_left_flag = 1; sl->merge_up_flag = 0; }
      }
    }
  }
  CTU_SYNC();
}

// ------------------------------------------------------------------------------------------------ real coder models
CTU_FN void enc_bin(const SmTables *T, uint8_t *ctx, int off, int val)
{
  const uint8_t st = ctx[off];
  ctx[off] = ((st & 1) == val) ? T->next_mps[st] : T->next_lps[st];
}

// All records and coefficients come from level 0 of the work tree: after the search it holds the CTU's decisions (the
// same values ctu_store wrote to the frame) and the border records of the left / above CTUs (ctu_load).
// The walk's state is the shared state block (re-derived with sm() in every function): the models in S->tmp, the
// records and coefficients in S->lv[0].
template <typename Pix> struct EncTrack { CtuST<Pix> *S; int x0, y0; };
template <typename Pix> CTU_FN const CuRec *tcu(const EncTrack<Pix> &e, int x, int y) { return cu_at(&e.S->lv[0], x - e.x0, y - e.y0); }

// encode_transform_coeff + encode_transform_unit (ref: encode_coding_tree.c:117-319), context-coded bins only
template <typename Pix> CTU_FN_NOINLINE void enc_transform_leaf(EncTrack<Pix> e, int x, int y, int depth, int tr_depth, int parent_u, int parent_v)
{
  CtuST<Pix> *S = e.S = sm(e.S);
  CabacState *cs = &S->tmp;
  const LcuLevel<Pix> *L0 = &S->lv[0];
  const CuRec *cur_pu = tcu(e, x, y);
  const CuRec *cur_cu = tcu(e, x & ~7, y & ~7);
  const int cb_y = cbf_is_set(cur_pu->cbf, depth, 0), cb_u = cbf_is_set(cur_cu->cbf, depth, 1), cb_v = cbf_is_set(cur_cu->cbf, depth, 2);
  if (depth < 4) {
    if (tr_depth == 0 || parent_u) enc_bin(&S->tb, cs->ctx, CTX_CBF_CHROMA + tr_depth, cb_u);
    if (tr_depth == 0 || parent_v) enc_bin(&S->tb, cs->ctx, CTX_CBF_CHROMA + tr_depth, cb_v);
  }
  enc_bin(&S->tb, cs->ctx, CTX_CBF_LUMA + (tr_depth ? 0 : 1), cb_y);        // CU_INTRA: always signalled
  if (!(cb_y | cb_u | cb_v)) return;
  const int width = 64 >> depth, width_c = depth == 4 ? width : width / 2;
  cs->update = 1;
  if (cb_y) {
    const int scan = scan_order_intra(cur_pu->mode, depth);
    coeff_cost_serial(&S->tb, &S->tb, &S->cfg, cs, L0->coeff_y + zorder(64, x & 63, y & 63), ilog2(width), 0, scan, cur_pu->tr_skip);
  }
  int xx = x, yy = y;
  if (depth == 4) {
    if (x % 8 == 0 || y % 8 == 0) return;
    xx -= 4; yy -= 4;
    cur_pu = tcu(e, xx, yy);
  }
  const int cu_u = cbf_is_set(cur_pu->cbf, depth, 1), cu_v = cbf_is_set(cur_pu->cbf, depth, 2);
  if (cu_u || cu_v) {
    const int scan = scan_order_intra(cur_pu->mode_chroma, depth);
    const int zi = zorder(32, (xx >> 1) & 31, (yy >> 1) & 31);
    if (cu_u) coeff_cost_serial(&S->tb, &S->tb, &S->cfg, cs, L0->coeff_u + zi, ilog2(width_c), 2, scan, 0);
    if (cu_v) coeff_cost_serial(&S->tb, &S->tb, &S->cfg, cs, L0->coeff_v + zi, ilog2(width_c), 2, scan, 0);
  }
}
template <typename Pix> CTU_FN void enc_transform_tree(const EncTrack<Pix> &e, int x, int y, int depth)
{
  // root of the CU's transform tree: tr_depth 0
  CtuST<Pix> *S = e.S;
  const CuRec *cur_cu = tcu(e, x & ~7, y & ~7);
  const int split = cur_cu->tr_depth > depth;
  if (!split) { enc_transform_leaf(e, x, y, depth, 0, 0, 0); return; }
  // one implicit split (64x64 CU into 32x32 TUs, or NxN into four 4x4 TUs)
  const int cb_u = cbf_is_set(cur_cu->cbf, depth, 1), cb_v = cbf_is_set(cur_cu->cbf, depth, 2);
  if (depth < 4) { enc_bin(&S->tb, S->tmp.ctx, CTX_CBF_CHROMA, cb_u); enc_bin(&S->tb, S->tmp.ctx, CTX_CBF_CHROMA, cb_v); }
  const int off = 64 >> (depth + 1);
  for (int k = 0; k < 4; ++k) enc_transform_leaf(e, x + (k & 1) * off, y + (k >> 1) * off, depth + 1, 1, cb_u, cb_v);
}

// one coding unit (no further split): part mode, intra modes, transform tree
template <typename Pix> CTU_FN_NOINLINE void enc_coding_unit(EncTrack<Pix> e, int x, int y, int depth)
{
  CtuST<Pix> *S = e.S = sm(e.S);
  uint8_t *ctx = S->tmp.ctx;
  const CuRec *cur_cu = tcu(e, x, y);
  const int cu_width = 64 >> depth;
  if (depth == 3) enc_bin(&S->tb, ctx, CTX_PART_SIZE, cur_cu->part_size == SIZE_2Nx2N ? 1 : 0);
  const int num_pu = cur_cu->part_size == SIZE_NxN ? 4 : 1;
  unsigned flag = 0;                // bit j: PU j's mode is an MPM
  int mode0 = 0;
  for (int j = 0; j < num_pu; ++j) {
    const int pw = cu_width / 2;
    const int pu_x = x + (num_pu == 4 ? (j & 1) * pw : 0), pu_y = y + (num_pu == 4 ? (j >> 1) * pw : 0);
    const CuRec *cur_pu = tcu(e, pu_x, pu_y);
    const CuRec *left_pu = pu_x > 0 ? tcu(e, pu_x - 1, pu_y) : NULL;
    const CuRec *above_pu = ((pu_y & 63) > 0 && pu_y > 0) ? tcu(e, pu_x, pu_y - 1) : NULL;
    int8_t preds[3];
    intra_mpm(pu_y, left_pu, above_pu, preds);
    if (j == 0) mode0 = cur_pu->mode;
    if (cur_pu->mode == preds[0] || cur_pu->mode == preds[1] || cur_pu->mode == preds[2]) flag |= 1u << j;
  }
  for (int j = 0; j < num_pu; ++j) enc_bin(&S->tb, ctx, CTX_INTRA_MODE, (flag >> j) & 1);
  enc_bin(&S->tb, ctx, CTX_CHROMA_PRED, cur_cu->mode_chroma == mode0 ? 0 : 1);
  enc_transform_tree(e, x, y, depth);
}

// kvz_encode_coding_tree: explicit traversal of the CU quadtree in coding order
template <typename Pix> CTU_FN_NOINLINE void enc_coding_tree(EncTrack<Pix> e)
{
  CtuST<Pix> *S = e.S = sm(e.S);
  const int Wd = S->cfg.width, H = S->cfg.height;
  // depth-first with a small stack of (x - x0) << 16 | (y - y0) << 8 | depth, at most 13 entries deep; it lives in the
  // rough search's SATD table, idle after the search
  int32_t *stk = S->satd;
  int sp = 1;
  stk[0] = 0;
  while (sp > 0) {
    --sp;
    const int v = stk[sp];
    const int x = e.x0 + (v >> 16), y = e.y0 + ((v >> 8) & 0xff), depth = v & 0xff;
    const CuRec *cur_cu = tcu(e, x, y);
    const int cu_width = 64 >> depth, half = cu_width >> 1;
    const int split_flag = cur_cu->depth > depth;
    const bool border_x = Wd < x + cu_width, border_y = H < y + cu_width;
    const bool border_split_x = Wd >= x + 8 + half, border_split_y = H >= y + 8 + half;
    const bool border = border_x || border_y;
    if (depth != 3) {
      if (!border) {
        int split_model = 0;
        if (x > 0 && tcu(e, x - 1, y)->depth > depth) ++split_model;
        if (y > 0 && tcu(e, x, y - 1)->depth > depth) ++split_model;
        enc_bin(&S->tb, S->tmp.ctx, CTX_SPLIT + split_model, split_flag);
      }
      if (split_flag || border) {
        // push in reverse so that the children pop in z-order
        const int c = v + 1;          // (x, y, depth + 1)
        if (!border || (border_split_x && border_split_y)) stk[sp++] = c + (half << 16) + (half << 8);
        if (!border_y || border_split_y) stk[sp++] = c + (half << 8);
        if (!border_x || border_split_x) stk[sp++] = c + (half << 16);
        stk[sp++] = c;
        continue;
      }
    }
    enc_coding_unit(e, x, y, depth);
  }
}

// The CTU's effect on the real coder's models; afterwards the row's state is published (and handed to the next row
// after the second CTU: WPP, encoderstate.c:759-771).  Leader only inside.
template <typename Pix> CTU_FN_NOINLINE void ctu_track_models(CtuST<Pix> *S, const FrameDevT<Pix> *F, int cx, int cy)
{
  S = sm(S);
  CTU_LEADER {
    // the models are walked in the search's spare copy (shared memory; the search is over): cost walks that adapt
    // them read and write shared memory, not the leader's stack
    CabacState &cs = S->tmp;
    cs = S->cabac0;
    cs.update = 1;
    if (S->cfg.sao_type) {
      const SaoRec *sl = &F->sao[2 * (cy * F->wlcu + cx)], *sc = sl + 1;
      if (cx > 0) enc_bin(&S->tb, cs.ctx, CTX_SAO_MERGE, sl->merge_left_flag);
      if (cy > 0 && !sl->merge_left_flag) enc_bin(&S->tb, cs.ctx, CTX_SAO_MERGE, sl->merge_up_flag);
      if (!sl->merge_left_flag && !sl->merge_up_flag) {
        enc_bin(&S->tb, cs.ctx, CTX_SAO_TYPE, sl->type != 0);
        enc_bin(&S->tb, cs.ctx, CTX_SAO_TYPE, sc->type != 0);
      }
    }
    const EncTrack<Pix> e = { S, cx * 64, cy * 64 };
    enc_coding_tree(e);
    cs.update = 0;
    F->row_ctx[cy] = cs;
    if (S->cfg.wpp && cx == 1 && cy + 1 < F->hlcu) F->row_ctx[cy + 1] = cs;
  }
  CTU_SYNC();
}

// ------------------------------------------------------------------------------------------------ whole CTU job
// The per-CTU functions find the configuration, the work area and the tables in the shared state block: they are
// copied there first.
template <typename Pix> CTU_FN void ctu_job(const CtxT<Pix> &c, const FrameDevT<Pix> *F, SaoStats *sao_scratch, int cx, int cy)
{
  CtuST<Pix> *S = sm(c.S);
  #pragma unroll 1
  for (int i = CTU_TID; i < (int)(sizeof(CtuConfig) / 4); i += CTU_NT) ((uint32_t *)&S->cfg)[i] = ((const uint32_t *)c.cfg)[i];
  CTU_LEADER S->W = c.W;
  CTU_SYNC();
  { PROF_T0(PR_LOAD); ctu_load(S, F, cx, cy); PROF_ADD(S, PR_LOAD); }
  { PROF_T0(PR_SEARCH); sm_tables_load(&S->tb, c.T); search_ctu(S, cx * 64, cy * 64); PROF_ADD(S, PR_SEARCH); }
  PROF_T0(PR_STORE);
  ctu_store(S, F, cx, cy);
#if defined(__CUDA_ARCH__)
  __threadfence();
#endif
  CTU_SYNC();
  PROF_ADD(S, PR_STORE);
  if (S->cfg.deblock_enable) { PROF_T0(PR_DEBLOCK); ctu_deblock(S, F, cx, cy); PROF_ADD(S, PR_DEBLOCK); }
  if (S->cfg.sao_type) { PROF_T0(PR_SAO); ctu_sao_search(S, F, sao_scratch, cx, cy); PROF_ADD(S, PR_SAO); }
  { PROF_T0(PR_TRACK); ctu_track_models(S, F, cx, cy); PROF_ADD(S, PR_TRACK); }
}

// ------------------------------------------------------------------------------------------------ SAO application
// Final picture of one CTU area from the deblocked planes (kvz_sao_reconstruct + sao_reconstruct_color semantics,
// sao.c:302-361, sao-generic.c:84-124): neighbours come from the deblocked picture, samples whose neighbour lies
// outside the picture keep their value.
template <typename Pix> CTU_FN_NOINLINE void ctu_sao_apply(const CtuConfig *cfg, const FrameDevT<Pix> *F, int cx, int cy)
{
  const int Wd = cfg->width, H = cfg->height;
  const SaoRec *sl = &F->sao[2 * (cy * F->wlcu + cx)], *sc = sl + 1;
  for (int plane = 0; plane < 3; ++plane) {
    const int sh = plane ? 1 : 0;
    const int pw = Wd >> sh, ph = H >> sh;
    const Pix *in = plane == 0 ? F->rec_y : (plane == 1 ? F->rec_u : F->rec_v);
    Pix *out = plane == 0 ? F->out_y : (plane == 1 ? F->out_u : F->out_v);
    const SaoRec *s = plane == 0 ? sl : sc;
    const int x0 = (cx * 64) >> sh, y0 = (cy * 64) >> sh;
    const int bw = imin(64 >> sh, pw - x0), bh = imin(64 >> sh, ph - y0);
    const int type = cfg->sao_type ? s->type : 0;
    const int ov = plane == 2 ? 5 : 0;
    #pragma unroll 1
    for (int e = CTU_TID; e < bw * bh; e += CTU_NT) {
      const int y = y0 + e / bw, x = x0 + e % bw;
      const int cc = in[(size_t)y * pw + x];
      int v = cc;
      if (type == 1) v = sao_band_px(cc, PixTraits<Pix>::bd, s->band_position[plane == 2 ? 1 : 0], s->offsets + ov);
      else if (type == 2) {
        int dx, dy;
        sao_eo_offsets(s->eo_class, dx, dy);
        const int xa = x + dx, ya = y + dy, xb = x - dx, yb = y - dy;
        if (xa >= 0 && xa < pw && xb >= 0 && xb < pw && ya >= 0 && ya < ph && yb >= 0 && yb < ph)
          v = sao_edge_px(cc, in[(size_t)ya * pw + xa], in[(size_t)yb * pw + xb], PixTraits<Pix>::bd, s->offsets + ov);
      }
      out[(size_t)y * pw + x] = (Pix)v;
    }
  }
}

}  // namespace kvzctu
