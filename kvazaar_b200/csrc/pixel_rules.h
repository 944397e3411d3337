// pixel_rules.h -- the reference's sample-domain rules, written once for every device path that predicts, deblocks or
// applies SAO: the strategy kernels (namespace kvzc), the CTU search driver (namespace kvzctu) and its host builds (g++,
// one-thread CTA).  Nothing here depends on how a caller's threads are arranged, where its samples live or how it loads
// them: the callers pass what they differ in (the samples already loaded, a pointer to the chosen reference row, an
// offset table).
//
//   * sample traits: the bit depth of a sample type and what follows from it;
//   * intra prediction: angular (displacement tables, projection of the side reference), planar, DC and filtered DC,
//     the mode 10 / 26 edge filter, when the smoothed references are used, the [1 2 1] reference smoothing;
//   * intra reference availability: the z-order rule of the available samples above / left of a 4x4 position, and the
//     counts of samples kvz_intra_build_reference copies;
//   * deblocking: beta, the tc table (a macro list), the 4-line luma filter and the chroma filter;
//   * SAO: the edge category, the neighbour offsets of an edge class, one sample filtered by a band or edge offset.
#pragma once
#include <stdint.h>
#include <type_traits>
#include "coeff_rules.h"

#if defined(__CUDACC__)
#define PIX_FN __device__ __forceinline__                   // rules only device code evaluates
#define PIX_HD __host__ __device__ __forceinline__          // rules the host also evaluates (table construction)
#define PIX_MFN __device__ __forceinline__                  // member functions of loaders
#else
#define PIX_FN static inline
#define PIX_HD static inline
#define PIX_MFN inline
#endif

// tc by Q (table 8-12 of the standard; kvz_g_tc_table_8x8, filter.c:60-66), indexed 0..53
#define PIX_DBK_TC \
  0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 1, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, \
  4, 5, 5, 6, 6, 7, 8, 9, 10, 11, 13, 14, 16, 18, 20, 22, 24

namespace kvzpix {

using kvzcoeff::iabs;
using kvzcoeff::imin;
PIX_HD int imax(int a, int b) { return a > b ? a : b; }
PIX_HD int iclip(int lo, int hi, int v) { return v < lo ? lo : (v > hi ? hi : v); }

// ---------------------------------------------------------------------------------------------- sample type
// The kernels are compiled once per sample type: uint8_t for 8-bit, uint16_t for 10-bit pictures (kvz_pixel of the
// reference's KVZ_BIT_DEPTH builds).  Everything that depends on the bit depth is derived from the type at compile time.
template <typename Pix> struct PixTraits {
  static_assert(std::is_same<Pix, uint8_t>::value || std::is_same<Pix, uint16_t>::value, "samples are uint8_t or uint16_t");
  static constexpr int bd = std::is_same<Pix, uint8_t>::value ? 8 : 10;
  static constexpr int max = (1 << bd) - 1;                           // CLIP_TO_PIXEL (ref: global.h)
  static constexpr int sao_max = (1 << ((bd < 10 ? bd : 10) - 5)) - 1;  // SAO_ABS_OFFSET_MAX (ref: global.h:230)
};

// ---------------------------------------------------------------------------------------------- intra prediction
// Reference arrays: index 0 = top-left corner sample, 1..2w along the edge (kvz_intra_references).
// The sample displacement and its inverse for an angular mode at |mode - 26| (vertical) / |10 - mode| (horizontal) =
// adisp, 0..8 (modedisp2sampledisp, modedisp2invsampledisp: intra-generic.c:59-60), as immediates packed into 64-bit
// words: a 9-entry array indexed at run time would be built in local memory on every use, inside the per-sample loops.
PIX_FN int ang_disp(int adisp)          // 0, 2, 5, 9, 13, 17, 21, 26, 32
{
  return adisp == 8 ? 32 : (int)((0x1A15110D09050200ull >> (8 * adisp)) & 0xff);
}
PIX_FN int ang_inv(int adisp)           // 0, 4096, 1638, 910, 630, 482, 390, 315, 256 = round(8192 / disp)
{
  if (adisp == 8) return 256;
  const uint64_t w = adisp < 4 ? 0x038E066610000000ull : 0x013B018601E20276ull;
  return (int)((w >> (16 * (adisp & 3))) & 0xffff);
}
// main-reference sample at block coordinate idx (>= -w .. 2w - 1); idx < -1 projects onto the side reference
// (intra-generic.c:88-108)
template <typename Pix> PIX_FN int ang_ref(const Pix *rmain, const Pix *rside, int idx, int inv)
{
  if (idx >= -1) return rmain[idx + 1];
  const int k = -idx - 1;
  return rside[(128 + k * inv) >> 8];
}
// one angular sample (mode 2..34) at output position (ox, oy) (intra-generic.c:49-155)
template <typename Pix> PIX_FN int angular_px(int mode, const Pix *top, const Pix *left, int ox, int oy)
{
  const bool vertical = mode >= 18;
  const int mdisp = vertical ? mode - 26 : 10 - mode;
  const int adisp = iabs(mdisp);
  const int sdisp = mdisp < 0 ? -ang_disp(adisp) : ang_disp(adisp);
  const Pix *rmain = vertical ? top : left;
  const Pix *rside = vertical ? left : top;
  const int x = vertical ? ox : oy, y = vertical ? oy : ox;
  if (sdisp == 0) return rmain[x + 1];
  const int pos = (y + 1) * sdisp;
  const int di = pos >> 5, df = pos & 31;
  const int inv = ang_inv(adisp);
  const int r1 = ang_ref(rmain, rside, x + di, inv);
  if (df == 0) return r1;
  const int r2 = ang_ref(rmain, rside, x + di + 1, inv);
  return ((32 - df) * r1 + df * r2 + 16) >> 5;
}
// planar (intra-generic.c:165-201)
template <typename Pix> PIX_FN int planar_px(int log2w, const Pix *top, const Pix *left, int x, int y)
{
  const int w = 1 << log2w;
  const int hor = (w - 1 - x) * left[y + 1] + (x + 1) * top[w + 1];
  const int ver = (w - 1 - y) * top[x + 1] + (y + 1) * left[w + 1];
  return (ver + hor + w) >> (log2w + 1);
}
// DC value of a block's references (intra-generic.c:210-241)
template <typename Pix> PIX_FN int dc_value(int log2w, const Pix *top, const Pix *left)
{
  const int w = 1 << log2w;
  int s = 0;
  for (int i = 1; i <= w; ++i) s += top[i] + left[i];
  return (s + w) >> (log2w + 1);
}
// DC with the first row and column filtered (luma below 32x32)
template <typename Pix> PIX_FN int filtered_dc_px(const Pix *top, const Pix *left, int dc, int x, int y)
{
  if (x == 0 && y == 0) return (left[1] + 2 * dc + top[1] + 2) >> 2;
  if (y == 0) return (top[x + 1] + 3 * dc + 2) >> 2;
  if (x == 0) return (left[y + 1] + 3 * dc + 2) >> 2;
  return dc;
}
// the edge filter of modes 10 / 26 on the first row / column: v plus half the gradient of the side reference
// (intra.c:207-219)
template <typename Pix> PIX_FN int intra_edge_px(int v, int side, int corner)
{
  return iclip(0, PixTraits<Pix>::max, v + ((side - corner) >> 1));
}
// should kvz_intra_predict use the smoothed references?  (intra.c:262-277)
PIX_FN bool intra_uses_filtered(int log2w, int mode, int color)
{
  if (color != 0 || mode == 1 || log2w == 2) return false;
  if (mode == 0) return true;
  const int thres = log2w == 3 ? 7 : (log2w == 4 ? 1 : 0);
  return imin(iabs(mode - 26), iabs(mode - 10)) > thres;
}
// kvz_intra_predict for one sample (intra.c:252-302).  r: the references, with members top, left, ftop, fleft (the
// smoothed ones, read only when intra_uses_filtered) and dc (dc_value of the unfiltered ones, read only for mode 1).
template <typename Pix, class R>
PIX_FN int intra_predict_px(const R &r, int log2w, int mode, int color, bool filter_boundary, int x, int y)
{
  const bool f = intra_uses_filtered(log2w, mode, color);
  const Pix *t = f ? r.ftop : r.top, *l = f ? r.fleft : r.left;
  if (mode == 0) return planar_px(log2w, t, l, x, y);
  if (mode == 1) return (color == 0 && log2w < 5) ? filtered_dc_px(t, l, (int)r.dc, x, y) : (int)r.dc;
  int v = angular_px(mode, t, l, x, y);
  if (color == 0 && log2w < 5 && filter_boundary) {
    if (mode == 10 && y == 0) v = intra_edge_px<Pix>(v, t[x + 1], t[0]);
    else if (mode == 26 && x == 0) v = intra_edge_px<Pix>(v, l[y + 1], l[0]);
  }
  return v;
}
// [1 2 1] smoothing of reference entry i of the top (is_top) or left edge, n = 2w + 1 entries (intra.c:176-204)
template <typename Pix> PIX_FN int ref_smooth_entry(const Pix *top, const Pix *left, bool is_top, int i, int n)
{
  if (i == 0) return (left[1] + 2 * left[0] + top[1] + 2) >> 2;
  const Pix *p = is_top ? top : left;
  if (i == n - 1) return p[i];
  return (p[i - 1] + 2 * p[i] + p[i + 1] + 2) >> 2;
}

// ---------------------------------------------------------------------------------------------- intra references
// Which reference samples the coding order has reconstructed (intra.c:47-82): a neighbouring 4x4 unit of the 64x64
// CTU is available when it comes earlier in z-order.  (ux, uy): 4x4 position in the CTU.
PIX_HD int zidx16(int ux, int uy)
{
  int z = 0;
  for (int b = 0; b < 4; ++b) z |= (((ux >> b) & 1) << (2 * b)) | (((uy >> b) & 1) << (2 * b + 1));
  return z;
}
// luma samples available above / left of the 4x4 unit at (ux, uy), inside the CTU's reach
PIX_HD int ref_px_top(int uy, int ux)
{
  if (uy == 0) return 64;
  const int z = zidx16(ux, uy);
  int n = 0;
  while (ux + n < 16 && zidx16(ux + n, uy - 1) < z) ++n;
  return 4 * n;
}
PIX_HD int ref_px_left(int uy, int ux)
{
  if (ux == 0) return 4 * (16 - uy);
  const int z = zidx16(ux, uy);
  int n = 0;
  while (uy + n < 16 && zidx16(ux - 1, uy + n) < z) ++n;
  return 4 * n;
}
// samples of one edge of a block of width w kvz_intra_build_reference finds available: the luma count of its 4x4
// position (ref_px_top / ref_px_left), in the colour's samples, at most the edge's 2w and what is left of the picture
// (`to_end`: luma samples from the block to the picture's right / bottom end)
PIX_FN int ref_avail(int luma_count, int is_c, int w, int to_end)
{
  int n = luma_count >> is_c;
  n = imin(n, 2 * w);
  return imin(n, to_end >> is_c);
}
// samples copied before the last one is replicated: the _inner variant (left and top both available) copies groups of
// four, at least one group (intra.c:486-494, 512-516)
PIX_FN int ref_copied(bool inner, int avail) { return inner ? imax(4, (avail + 3) & ~3) : avail; }

// ---------------------------------------------------------------------------------------------- deblocking
// beta by Q (table 8-12; kvz_g_beta_table_8x8, filter.c:48-58), Q = 0..51
PIX_FN int dbk_beta(int i) { return i < 16 ? 0 : (i < 29 ? i - 10 : 2 * i - 38); }

// How the filters read the samples around an edge: plain loads here; a caller whose samples need other loads passes its
// own loader (the CTU search reads frame samples written by other CTAs through L2).
struct PlainLoad { template <typename Pix> PIX_MFN int operator()(const Pix *p) const { return *p; } };

// The luma filter of one 4-line part (filter.c:95-170, 474-520): px -> q0 of line 0, xs across the edge, ys along it.
// Decides and writes the filtered samples.
template <typename Pix, typename S, class Ld = PlainLoad>
PIX_FN void dbk_luma_part(Pix *px, S xs, S ys, int beta, int tc, Ld ld = Ld())
{
  int b[4][8];                      // b[l][i]: sample i - 4 across the edge of line l
  for (int l = 0; l < 4; ++l) for (int i = 0; i < 8; ++i) b[l][i] = ld(&px[l * ys + (i - 4) * xs]);
  const int dp0 = iabs(b[0][1] - 2 * b[0][2] + b[0][3]), dq0 = iabs(b[0][4] - 2 * b[0][5] + b[0][6]);
  const int dp3 = iabs(b[3][1] - 2 * b[3][2] + b[3][3]), dq3 = iabs(b[3][4] - 2 * b[3][5] + b[3][6]);
  const int dp = dp0 + dp3, dq = dq0 + dq3;
  if (dp + dq >= beta) return;
  const bool strong = 2 * (dp0 + dq0) < (beta >> 2) && 2 * (dp3 + dq3) < (beta >> 2) &&
                      iabs(b[0][3] - b[0][4]) < ((5 * tc + 1) >> 1) && iabs(b[3][3] - b[3][4]) < ((5 * tc + 1) >> 1) &&
                      iabs(b[0][0] - b[0][3]) + iabs(b[0][4] - b[0][7]) < (beta >> 3) &&
                      iabs(b[3][0] - b[3][3]) + iabs(b[3][4] - b[3][7]) < (beta >> 3);
  const int side = (beta + (beta >> 1)) >> 3;
  for (int l = 0; l < 4; ++l) {
    const int m0 = b[l][0], m1 = b[l][1], m2 = b[l][2], m3 = b[l][3], m4 = b[l][4], m5 = b[l][5], m6 = b[l][6], m7 = b[l][7];
    Pix *row = px + l * ys;
    if (strong) {
      row[-3 * xs] = (Pix)iclip(m1 - 2 * tc, m1 + 2 * tc, (2 * m0 + 3 * m1 + m2 + m3 + m4 + 4) >> 3);
      row[-2 * xs] = (Pix)iclip(m2 - 2 * tc, m2 + 2 * tc, (m1 + m2 + m3 + m4 + 2) >> 2);
      row[-1 * xs] = (Pix)iclip(m3 - 2 * tc, m3 + 2 * tc, (m1 + 2 * m2 + 2 * m3 + 2 * m4 + m5 + 4) >> 3);
      row[0] = (Pix)iclip(m4 - 2 * tc, m4 + 2 * tc, (m2 + 2 * m3 + 2 * m4 + 2 * m5 + m6 + 4) >> 3);
      row[xs] = (Pix)iclip(m5 - 2 * tc, m5 + 2 * tc, (m3 + m4 + m5 + m6 + 2) >> 2);
      row[2 * xs] = (Pix)iclip(m6 - 2 * tc, m6 + 2 * tc, (m3 + m4 + m5 + 3 * m6 + 2 * m7 + 4) >> 3);
    } else {
      int delta = (9 * (m4 - m3) - 3 * (m5 - m2) + 8) >> 4;
      if (iabs(delta) < tc * 10) {
        delta = iclip(-tc, tc, delta);
        row[-1 * xs] = (Pix)iclip(0, PixTraits<Pix>::max, m3 + delta);
        row[0] = (Pix)iclip(0, PixTraits<Pix>::max, m4 - delta);
        if (dp < side) row[-2 * xs] = (Pix)iclip(0, PixTraits<Pix>::max, m2 + iclip(-(tc >> 1), tc >> 1, (((m1 + m3 + 1) >> 1) - m2 + delta) >> 1));
        if (dq < side) row[xs] = (Pix)iclip(0, PixTraits<Pix>::max, m5 + iclip(-(tc >> 1), tc >> 1, (((m6 + m4 + 1) >> 1) - m5 - delta) >> 1));
      }
    }
  }
}
// The chroma filter of one 4-line part (filter.c:175-192): px -> q0 of line 0, xs across the edge, ys along it.
// Writes p0 and q0 of every line.
template <typename Pix, typename S, class Ld = PlainLoad>
PIX_FN void dbk_chroma_part(Pix *px, S xs, S ys, int tc, Ld ld = Ld())
{
  for (int l = 0; l < 4; ++l) {
    Pix *s = px + l * ys;
    const int m2 = ld(&s[-2 * xs]), m3 = ld(&s[-xs]), m4 = ld(&s[0]), m5 = ld(&s[xs]);
    const int delta = iclip(-tc, tc, (((m4 - m3) * 4) + m2 - m5 + 4) >> 3);
    s[-xs] = (Pix)iclip(0, PixTraits<Pix>::max, m3 + delta);
    s[0] = (Pix)iclip(0, PixTraits<Pix>::max, m4 - delta);
  }
}

// ---------------------------------------------------------------------------------------------- SAO
// edge category of sample c between its neighbours a and b (sao_shared_generics.h:41-50): idx = 2 + sign(c - a) +
// sign(c - b) -> { 1, 2, 0, 3, 4 }, packed four bits per entry
PIX_FN int sao_eo_cat(int a, int b, int c)
{
  const int idx = 2 + ((c > a) - (c < a)) + ((c > b) - (c < b));
  return (0x43021 >> (4 * idx)) & 7;
}
// neighbour a of edge class eo at (ax, ay) from the sample; neighbour b is at (-ax, -ay) (sao.h:71-76)
PIX_FN void sao_eo_offsets(int eo, int &ax, int &ay)
{
  ax = (eo == 1) ? 0 : (eo == 3 ? 1 : -1);
  ay = (eo == 0) ? 0 : -1;
}
// one sample v filtered by the band offsets of a plane (sao-generic.c:84-124 with the band table of
// kvz_calc_sao_offset_array, sao.c:180-202): offs[1..4] belong to the bands band_pos .. band_pos + 3
template <class Off> PIX_FN int sao_band_px(int v, int bitdepth, int band_pos, const Off &offs)
{
  const int k = (v >> (bitdepth - 5)) - band_pos;
  return (k >= 0 && k <= 3) ? iclip(0, (1 << bitdepth) - 1, v + offs[k + 1]) : v;
}
// one sample v between neighbours a and b filtered by the edge offsets of a plane: offs[category]
template <class Off> PIX_FN int sao_edge_px(int v, int a, int b, int bitdepth, const Off &offs)
{
  return iclip(0, (1 << bitdepth) - 1, v + offs[sao_eo_cat(a, b, v)]);
}

}  // namespace kvzpix
