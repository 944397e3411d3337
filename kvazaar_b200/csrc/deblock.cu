// deblock.cu -- frame-level HEVC deblocking filter (SURVEY §8f rank 3; ref: src/filter.c:95-792).
//
// The reference filters LCU by LCU inside the CTU job (kvz_filter_deblock_lcu, filter.c:783-792), delaying the
// rightmost four columns of horizontal edges so that they only see vertically filtered columns.  Per frame that is
// the standard two passes: all vertical edges of the 8x8 grid, then all horizontal edges on the result.  Here each
// pass is ONE launch over the three planes; a thread owns one 4-sample edge part (blockIdx.y: luma, U, V), consecutive
// threads walk along the row so that every row access of a warp is one contiguous 128/256-byte run.
//
// Edges are independent inside a pass: a part reads 4 samples and writes at most 3 on either side of an edge of
// the 8-sample grid, so no two parts of the same pass touch a common sample.  The passes run in place.
//
// Decision inputs are the reference's own per-SCU records (cu_info_t memory image, 20 B per 4x4, src/cu.h:126-165):
// the binding uploads frame->cu_array->data as it is.
#include "common.cuh"

namespace kvzc {

__constant__ uint8_t c_dbk_tc[54] = { PIX_DBK_TC };

struct DbkCu {
  uint32_t w0, w1, mv0, mv1, w4;
  __device__ int type() const { return w0 & 3; }
  __device__ int depth() const { return (w0 >> 2) & 7; }
  __device__ int part_size() const { return (w0 >> 5) & 7; }
  __device__ int tr_depth() const { return (w0 >> 8) & 7; }
  __device__ int cbf() const { return w1 & 0xffff; }
  __device__ int qp() const { return (w1 >> 16) & 0xff; }
  __device__ int mvx(int l) const { return (int16_t)((l ? mv1 : mv0) & 0xffff); }
  __device__ int mvy(int l) const { return (int16_t)((l ? mv1 : mv0) >> 16); }
  __device__ int mv_ref(int l) const { return (w4 >> (8 * l)) & 0xff; }
  __device__ int mv_dir() const { return (w4 >> 22) & 3; }
  __device__ bool cbf_y() const { const int m[5] = { 0x1f, 0x0f, 0x07, 0x03, 0x01 }; return (cbf() & m[min(tr_depth(), 4)]) != 0; }
};

__device__ __forceinline__ DbkCu dbk_cu_at(const uint32_t *__restrict__ cus, int stride_scu, int x, int y)
{
  const uint32_t *r = cus + 5 * ((size_t)(x >> 2) + (size_t)(y >> 2) * stride_scu);
  DbkCu c;
  c.w0 = r[0]; c.w1 = r[1]; c.mv0 = r[2]; c.mv1 = r[3]; c.w4 = r[4];
  return c;
}

// is the left (top) edge of the 8x8 unit at (x, y) a TU or PU boundary?  (filter.c:194-246)
__device__ __forceinline__ bool dbk_edge_wanted(const uint32_t *cus, int stride_scu, int x, int y, bool hor, bool &tu_boundary)
{
  const DbkCu s = dbk_cu_at(cus, stride_scu, x, y);
  const int tu_w = 64 >> s.tr_depth(), cu_w = 64 >> s.depth();
  const int pos = hor ? y : x;
  tu_boundary = (pos & (tu_w - 1)) == 0;
  if (tu_boundary) return true;
  const DbkCu cu = dbk_cu_at(cus, stride_scu, x & ~(cu_w - 1), y & ~(cu_w - 1));
  const int cu_pos = pos & ~(cu_w - 1);
  // quarter position of the second PU along this axis per part mode (kvz_part_mode_offsets, cu.c:63-72)
  const int q = ((hor ? 0x00312020u : 0x31002200u) >> (4 * cu.part_size())) & 0xf;
  return pos == cu_pos || (q != 0 && pos == cu_pos + q * cu_w / 4);
}

__device__ __forceinline__ bool dbk_far(int ax, int ay, int bx, int by) { return abs(ax - bx) >= 4 || abs(ay - by) >= 4; }

// boundary strength of one 4-sample part (filter.c:385-470)
__device__ __forceinline__ int dbk_strength(const kvz_cuda_dbk_params &p, const DbkCu &P, const DbkCu &Q, bool tu_boundary)
{
  if (Q.type() == 1 || P.type() == 1) return 2;
  if (tu_boundary && (Q.cbf_y() || P.cbf_y())) return 1;
  const int dp = P.mv_dir(), dq = Q.mv_dir();
  if (dp != 3 && dq != 3) {
    const int lp = (dp - 1) & 1, lq = (dq - 1) & 1;
    if (dbk_far(Q.mvx(lq), Q.mvy(lq), P.mvx(lp), P.mvy(lp))) return 1;
    if (Q.mv_ref(lq) != P.mv_ref(lp)) return 1;
  }
  if (!p.slice_is_b) return 0;
  const int p0x = (dp & 1) ? P.mvx(0) : 0, p0y = (dp & 1) ? P.mvy(0) : 0, p1x = (dp & 2) ? P.mvx(1) : 0, p1y = (dp & 2) ? P.mvy(1) : 0;
  const int q0x = (dq & 1) ? Q.mvx(0) : 0, q0y = (dq & 1) ? Q.mvy(0) : 0, q1x = (dq & 2) ? Q.mvx(1) : 0, q1y = (dq & 2) ? Q.mvy(1) : 0;
  const int rp0 = (dp & 1) ? p.ref_LX[0][P.mv_ref(0) & 15] : -1, rp1 = (dp & 2) ? p.ref_LX[1][P.mv_ref(1) & 15] : -1;
  const int rq0 = (dq & 1) ? p.ref_LX[0][Q.mv_ref(0) & 15] : -1, rq1 = (dq & 2) ? p.ref_LX[1][Q.mv_ref(1) & 15] : -1;
  if (!((rp0 == rq0 && rp1 == rq1) || (rp0 == rq1 && rp1 == rq0))) return 1;
  const bool straight = dbk_far(q0x, q0y, p0x, p0y) || dbk_far(q1x, q1y, p1x, p1y);
  const bool crossed = dbk_far(q1x, q1y, p0x, p0y) || dbk_far(q0x, q0y, p1x, p1y);
  if (rp0 != rp1) return rp0 == rq0 ? straight : crossed;
  return straight && crossed;
}

__device__ __forceinline__ int dbk_qp(const kvz_cuda_dbk_params &p, const uint32_t *cus, int x, int y, bool hor)
{
  if (!p.per_cu_qp) return p.qp;
  const int qp_p = hor ? dbk_cu_at(cus, p.cu_stride_scu, x, y - 1).qp() : dbk_cu_at(cus, p.cu_stride_scu, x - 1, y).qp();
  return (qp_p + dbk_cu_at(cus, p.cu_stride_scu, x, y).qp() + 1) >> 1;
}

// One pass (HOR = false: vertical edges, true: horizontal edges).  blockIdx.y = plane.
//   luma   : parts indexed (along-edge 4-sample index, edge index); thread order follows the sample rows
//   chroma : one part per 8x8 luma unit whose edge coordinate is a multiple of 16
template <class T, bool HOR>
__global__ void __launch_bounds__(128) deblock_pass_kernel(kvz_cuda_dbk_params p, T *__restrict__ y, T *__restrict__ u, T *__restrict__ v,
                                                           const uint32_t *__restrict__ cus)
{
  const int W = p.width, H = p.height;
  const int scale = 1 << (PixTraits<T>::bd - 8);
  const int plane = blockIdx.y;
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (plane == 0) {
    // HOR: t -> (px / 4 fastest, edge row ey = 8 * (1 + t / (W / 4)));  VER: t -> (edge ex = 8 * (1 + t % (W / 8 - 1)) fastest, py / 4)
    int px, py;
    if (HOR) { const int per_row = W / 4; px = (t % per_row) * 4; py = (1 + t / per_row) * 8; }
    else { const int per_row = W / 8 - 1; if (per_row <= 0) return; px = (1 + t % per_row) * 8; py = (t / per_row) * 4; }
    if (px >= W || py >= H) return;
    const int ux = HOR ? (px & ~7) : px, uy = HOR ? py : (py & ~7);             // the 8x8 unit this part belongs to
    bool tu_boundary;
    if (!dbk_edge_wanted(cus, p.cu_stride_scu, ux, uy, HOR, tu_boundary)) return;
    const DbkCu Q = dbk_cu_at(cus, p.cu_stride_scu, px, py), P = dbk_cu_at(cus, p.cu_stride_scu, HOR ? px : px - 1, HOR ? py - 1 : py);
    const int bs = dbk_strength(p, P, Q, tu_boundary);
    if (!bs) return;
    const int qp = dbk_qp(p, cus, ux, uy, HOR);
    const int beta = dbk_beta(clip3(0, 51, qp + 2 * p.beta_offset_div2)) * scale;
    const int tc = c_dbk_tc[clip3(0, 53, qp + 2 * (bs - 1) + 2 * p.tc_offset_div2)] * scale;
    dbk_luma_part<T, long>(y + (size_t)py * W + px, HOR ? W : 1, HOR ? 1 : W, beta, tc);
  } else {
    if (!u || !v) return;
    const int Wc = W / 2, Hc = H / 2;
    // units: edge coordinate multiple of 16 luma samples; the other coordinate steps by 8 luma samples
    int ex, ey;
    if (HOR) { const int per_row = W / 8; ex = (t % per_row) * 8; ey = (1 + t / per_row) * 16; }
    else { const int per_row = (W - 1) / 16; if (per_row <= 0) return; ex = (1 + t % per_row) * 16; ey = (t / per_row) * 8; }
    if (ex >= W || ey >= H) return;
    const DbkCu Q = dbk_cu_at(cus, p.cu_stride_scu, ex, ey), P = dbk_cu_at(cus, p.cu_stride_scu, HOR ? ex : ex - 2, HOR ? ey - 2 : ey);
    if (Q.type() != 1 && P.type() != 1) return;
    bool tu_boundary;
    if (!dbk_edge_wanted(cus, p.cu_stride_scu, ex, ey, HOR, tu_boundary)) return;
    const int cx = ex / 2, cy = ey / 2;
    if (cx >= Wc || cy >= Hc) return;
    const int qpc = kvzcoeff::scaled_qp(2, dbk_qp(p, cus, ex, ey, HOR), 0);       // kvz_g_chroma_scale (filter.c:589)
    const int tc = c_dbk_tc[clip3(0, 53, qpc + 2 + 2 * p.tc_offset_div2)] * scale;
    T *pl = plane == 1 ? u : v;
    dbk_chroma_part<T, long>(pl + (size_t)cy * Wc + cx, HOR ? Wc : 1, HOR ? 1 : Wc, tc);
  }
}

template <class T>
static int deblock_launch(const kvz_cuda_dbk_params &p, T *y, T *u, T *v, const uint32_t *cus, cudaStream_t st)
{
  const int W = p.width, H = p.height;
  // vertical edges: luma (W/8 - 1) x (H/4) parts, chroma ((W-1)/16) x (H/8)
  {
    const long luma = (long)(W / 8 - 1) * (H / 4), chroma = (long)((W - 1) / 16) * (H / 8);
    const long n = luma > chroma ? luma : chroma;
    if (n > 0) {
      deblock_pass_kernel<T, false><<<dim3((unsigned)((n + 127) / 128), 3), 128, 0, st>>>(p, y, u, v, cus);
      KVZC_LAUNCHED();
    }
  }
  // horizontal edges: luma (W/4) x (H/8 - 1), chroma (W/8) x ((H-1)/16)
  {
    const long luma = (long)(W / 4) * (H / 8 - 1), chroma = (long)(W / 8) * ((H - 1) / 16);
    const long n = luma > chroma ? luma : chroma;
    if (n > 0) {
      deblock_pass_kernel<T, true><<<dim3((unsigned)((n + 127) / 128), 3), 128, 0, st>>>(p, y, u, v, cus);
      KVZC_LAUNCHED();
    }
  }
  return 0;
}

}  // namespace kvzc

using namespace kvzc;

extern "C" {

int kvz_cuda_deblock_frame(const kvz_cuda_dbk_params *p, int bitdepth, void *y_dev, void *u_dev, void *v_dev, const void *cus_dev, void *stream)
{
  KVZC_REQUIRE_DEVICE();
  KVZC_ARG(p && y_dev && cus_dev && (bitdepth == 8 || bitdepth == 10));
  KVZC_ARG(p->width >= 8 && p->height >= 8 && p->width % 8 == 0 && p->height % 8 == 0 && p->cu_stride_scu >= p->width / 4);
  KVZC_ARG((u_dev == nullptr) == (v_dev == nullptr));
  if (bitdepth == 8) return deblock_launch<uint8_t>(*p, (uint8_t *)y_dev, (uint8_t *)u_dev, (uint8_t *)v_dev, (const uint32_t *)cus_dev, as_stream(stream));
  return deblock_launch<uint16_t>(*p, (uint16_t *)y_dev, (uint16_t *)u_dev, (uint16_t *)v_dev, (const uint32_t *)cus_dev, as_stream(stream));
}

// Host-buffer form for the binding (INTEGRATION.md "deblocking"): planes with their own strides, cu_info_t array as
// the reference holds it.  Synchronous; uses the calling thread's staging buffers and stream.
int kvz_cuda_call_deblock_frame(const kvz_cuda_dbk_params *p, int bitdepth, void *y, void *u, void *v, int stride, const void *cus)
{
  KVZC_REQUIRE_DEVICE();
  KVZC_ARG(p && y && u && v && cus && (bitdepth == 8 || bitdepth == 10) && stride >= p->width);
  const size_t px = bitdepth == 8 ? 1 : 2;
  const int W = p->width, H = p->height, Wc = W / 2, Hc = H / 2;
  const size_t ybytes = (size_t)W * H * px, cbytes = (size_t)Wc * Hc * px;
  const size_t cu_rows = (size_t)(H + 3) / 4, cubytes = cu_rows * p->cu_stride_scu * 20;
  Call c(ybytes + 2 * cbytes + cubytes + 4096);
  KVZC_ARG(c.ok);
  uint8_t *dy = c.in2d((const uint8_t *)y, (int)(W * px), H, (long)stride * px);
  uint8_t *du = c.in2d((const uint8_t *)u, (int)(Wc * px), Hc, (long)(stride / 2) * px);
  uint8_t *dv = c.in2d((const uint8_t *)v, (int)(Wc * px), Hc, (long)(stride / 2) * px);
  const uint8_t *dcu = c.in((const uint8_t *)cus, cubytes);
  if (int r = c.upload()) return r;
  if (int r = kvz_cuda_deblock_frame(p, bitdepth, dy, du, dv, dcu, c.s.stream)) return r;
  // planes come back in place: download the input region that holds them
  KVZC_CHECK(cudaMemcpyAsync(c.s.h, c.s.d, (size_t)((uint8_t *)dcu - c.s.d), cudaMemcpyDeviceToHost, c.s.stream));
  KVZC_CHECK(cudaStreamSynchronize(c.s.stream));
  const uint8_t *hy = c.host_ptr(dy), *hu = c.host_ptr(du), *hv = c.host_ptr(dv);
  for (int r = 0; r < H; ++r) memcpy((uint8_t *)y + (size_t)r * stride * px, hy + (size_t)r * W * px, (size_t)W * px);
  for (int r = 0; r < Hc; ++r) {
    memcpy((uint8_t *)u + (size_t)r * (stride / 2) * px, hu + (size_t)r * Wc * px, (size_t)Wc * px);
    memcpy((uint8_t *)v + (size_t)r * (stride / 2) * px, hv + (size_t)r * Wc * px, (size_t)Wc * px);
  }
  return 0;
}

}  // extern "C"
