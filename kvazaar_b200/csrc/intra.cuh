// intra.cuh -- intra prediction device primitives of the strategy kernels.
// The prediction rules themselves (angular, planar, DC, the edge filter, reference smoothing and availability) are
// in pixel_rules.h, shared with the CTU search.  Every prediction sample has a closed form in the reference samples,
// so each thread computes its own pixels directly -- no sequential accumulation, no transposition pass.  Here: the
// reference build of kvz_intra_build_reference (ref: src/intra.c:305-559) over a frame plane.
#pragma once
#include "common.cuh"

namespace kvzc {

// the references of one block as intra_predict_px reads them (pixel_rules.h)
template <class T> struct RefView {
  const T *top, *left;      // unfiltered
  const T *ftop, *fleft;    // [1 2 1]-smoothed (only read where intra_uses_filtered)
  int dc;                   // dc_value of the unfiltered references
};

// Per-block constants of kvz_intra_build_reference over a frame plane
struct BuildRefCtx {
  int px, py;           // plane coordinates of the block
  int n_left, n_top;    // number of samples copied before the last one is replicated (0 = edge fill)
  bool inner, has_left, has_top;
};
__device__ __forceinline__ BuildRefCtx build_ref_ctx(int log2w, int color, int luma_x, int luma_y, int pic_w, int pic_h)
{
  BuildRefCtx c;
  const int is_c = color != 0, w = 1 << log2w;
  const int lx = luma_x & 63, ly = luma_y & 63;
  c.px = luma_x >> is_c; c.py = luma_y >> is_c;
  c.has_left = luma_x > 0; c.has_top = luma_y > 0;
  c.inner = c.has_left && c.has_top;
  const int al = c.has_left ? ref_avail(ref_px_left(ly >> 2, lx >> 2), is_c, w, pic_h - luma_y) : 0;
  const int at = c.has_top ? ref_avail(ref_px_top(ly >> 2, lx >> 2), is_c, w, pic_w - luma_x) : 0;
  c.n_left = ref_copied(c.inner, al);
  c.n_top = ref_copied(c.inner, at);
  return c;
}
// entry i (0 = corner, 1..2w) of the left / top reference
template <class T>
__device__ __forceinline__ int build_ref_entry(const BuildRefCtx &c, const T *rec, int stride, bool is_top, int i)
{
  constexpr int DC = 1 << (PixTraits<T>::bd - 1);
#define KVZC_REC(xx, yy) ((int)rec[(long)(yy) * stride + (xx)])
  // left[1] is needed for the non-inner corner
  auto left_at = [&](int k) -> int {   // k = 0..2w-1
    if (c.has_left) return KVZC_REC(c.px - 1, c.py + min(k, c.n_left - 1));
    return c.has_top ? KVZC_REC(c.px, c.py - 1) : DC;
  };
  if (i == 0) return c.inner ? KVZC_REC(c.px - 1, c.py - 1) : left_at(0);
  if (!is_top) return left_at(i - 1);
  if (c.has_top) return KVZC_REC(c.px + min(i - 1, c.n_top - 1), c.py - 1);
  return c.has_left ? KVZC_REC(c.px - 1, c.py) : DC;
#undef KVZC_REC
}

}  // namespace kvzc
