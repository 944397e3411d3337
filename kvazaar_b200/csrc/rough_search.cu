// rough_search.cu -- fused frame-level rough intra search (the dominant kernel of the frame pass), 8- and 10-bit samples.
//
// Per W x W luma block: reference samples (kvz_intra_build_reference over the reconstruction plane) -> [1 2 1]
// smoothing -> all 35 kvz_intra_predict modes -> satd_WxW against the source.  (search_intra_rough's inner loop,
// ref: search_intra.c:391-530, intra.c:176-302, intra-generic.c, picture-generic.c:252-340.)
//
// Mapping (chosen for the SIMT machine, not the reference's loop order):
//   * a CTA owns 32 8x8 sub-blocks (32 blocks of 8x8, 8 of 16x16, 2 of 32x32; 4x4: 32 blocks); lane = sub-block;
//   * each of the 4 warps walks its own subset of the 35 modes, so the mode -- and with it the projection
//     direction, the per-row displacement, the reference selection -- is WARP-UNIFORM: no divergence;
//   * a thread never materialises pixels: for each row it loads a 9-byte window of the (extended) main reference
//     from shared memory, builds the (col c, col c+2) 16-bit lane pairs the packed Hadamard wants directly
//     with PRMT, interpolates two samples per IMAD pair, and subtracts from the source lanes kept in registers
//     (the source block and its transpose are packed once and reused for all modes);
//   * horizontal modes (2..17) are evaluated in the transposed domain against the transposed source: SATD is
//     invariant under transposition, so the reference's final transpose pass disappears;
//   * df == 0 needs no branch: ((32-0)*a + 0*b + 16) >> 5 == a;
//   * 16-bit samples (10-bit video) take the same walk: a 32-bit word already holds two samples, the (c, c+2) lane
//     pairs come from PRMT over neighbouring words, two interpolations per IMAD pair still fit (32 * 1023 + 16 < 2^16),
//     and the packed Hadamard stays exact: five butterfly stages of |d| <= 1023 reach 32736 < 2^15, the sixth is the
//     2 * max(|lo|, |hi|) fold.
// HBM traffic per block: W*W source + (4W+1) reference samples in, 35 costs out.
#include "common.cuh"
#include "intra.cuh"
#include "satd.cuh"

namespace kvzc {

template <class T>
__device__ __forceinline__ uint32_t interp2(uint32_t a, uint32_t b, uint32_t f0, uint32_t f1)
{
  constexpr uint32_t MASK = ((1u << PixTraits<T>::bd) - 1u) * 0x00010001u;
  return ((a * f0 + b * f1 + 0x00100010u) >> 5) & MASK;           // two samples: ((32-f)*a + f*b + 16) >> 5
}

template <class T, int LOG2W>
__global__ void __launch_bounds__(128) rough_search_u8_kernel(const T *__restrict__ src, const T *__restrict__ rec,
                                                              int stride, int pic_w, int pic_h, int blocks_x, int nblk,
                                                              uint32_t *__restrict__ costs, int8_t *__restrict__ best_mode,
                                                              uint32_t *__restrict__ best_cost)
{
  constexpr int W = 1 << LOG2W;
  constexpr int S = W >= 8 ? W / 8 : 1, SUBS = S * S, GROUP = 32 / SUBS;
  constexpr int N = 2 * W + 1;
  constexpr int RS = ((N + 3) / 4) * 4;                          // 12, 20, 36, 68 bytes: odd word stride
  constexpr int EN = 3 * W + 1;
  constexpr int ES = W == 4 ? 20 : ((EN + 3) / 4) * 4;           // 20, 28, 52, 100 bytes: odd word stride
  constexpr int R = W >= 8 ? 8 : 4;                              // rows / cols of a lane's sub-block
  constexpr int K = R / 2;                                       // packed lane registers per row
  constexpr bool WIDE = sizeof(T) == 2;                          // 16-bit samples
  __shared__ __align__(16) T s_ref[GROUP][4][RS];                // top, left, smoothed top, smoothed left
  __shared__ __align__(16) T s_plain[GROUP][4][ES];              // same, shifted so that index j = idx + W
  __shared__ __align__(16) T s_ext[4][GROUP][ES];                // per-warp scratch: main ref with projected side part
  __shared__ int s_dc[GROUP];
  __shared__ BuildRefCtx s_ctx[GROUP];
  __shared__ uint32_t s_cost[GROUP][36];                         // per-block cost table for the fused mode selection

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int first = blockIdx.x * GROUP;
  const int g = lane / SUBS, sub = lane % SUBS;
  const int sy = sub / S, sx = sub % S;
  const int blk = first + g;
  const bool valid = blk < nblk;

  // ---- reference samples for the GROUP blocks (all 128 threads)
  if (threadIdx.x < GROUP) {
    const int b = min(first + (int)threadIdx.x, nblk - 1);
    s_ctx[threadIdx.x] = build_ref_ctx(LOG2W, 0, (b % blocks_x) * W, (b / blocks_x) * W, pic_w, pic_h);
  }
  __syncthreads();
  for (int e = threadIdx.x; e < GROUP * 2 * N; e += 128) {
    const int gb = e / (2 * N), r = e - gb * 2 * N;
    const bool is_top = r < N;
    const int k = is_top ? r : r - N;
    s_ref[gb][is_top ? 0 : 1][k] = (T)build_ref_entry(s_ctx[gb], rec, stride, is_top, k);
  }
  __syncthreads();
  for (int e = threadIdx.x; e < GROUP * 2 * N; e += 128) {
    const int gb = e / (2 * N), r = e - gb * 2 * N;
    const bool is_top = r < N;
    const int k = is_top ? r : r - N;
    s_ref[gb][is_top ? 2 : 3][k] = (T)ref_smooth_entry(s_ref[gb][0], s_ref[gb][1], is_top, k, N);
  }
  if (threadIdx.x < GROUP) s_dc[threadIdx.x] = dc_value(LOG2W, s_ref[threadIdx.x][0], s_ref[threadIdx.x][1]);
  __syncthreads();
  for (int e = threadIdx.x; e < GROUP * 4 * ES; e += 128) {
    const int gb = e / (4 * ES), r = e - gb * 4 * ES, a = r / ES, j = r - a * ES;
    const int idx = j - W;                                       // block coordinate of entry j
    s_plain[gb][a][j] = (idx >= -1 && idx + 1 < N) ? s_ref[gb][a][idx + 1] : 0;
  }
  __syncthreads();

  // ---- source lanes of this lane's sub-block: SA (as is) and ST (transposed), packed (c, c+2) pairs
  uint32_t SA[R][K], ST[R][K];
  if constexpr (WIDE) {
    // 16-bit samples: row r = R / 2 words of two samples each
    uint32_t rows[R][R / 2];
    const int bx = valid ? blk % blocks_x : 0, by = valid ? blk / blocks_x : 0;
    const T *p = src + (long)(by * W + sy * R) * stride + bx * W + sx * R;
#pragma unroll
    for (int r = 0; r < R; ++r) {
      if constexpr (R == 8) {
        const uint4 v = valid ? __ldg(reinterpret_cast<const uint4 *>(p + (long)r * stride)) : make_uint4(0, 0, 0, 0);
        rows[r][0] = v.x; rows[r][1] = v.y; rows[r][2] = v.z; rows[r][3] = v.w;
      } else {
        const uint2 v = valid ? __ldg(reinterpret_cast<const uint2 *>(p + (long)r * stride)) : make_uint2(0, 0);
        rows[r][0] = v.x; rows[r][1] = v.y;
      }
    }
#pragma unroll
    for (int r = 0; r < R; ++r)
#pragma unroll
      for (int h = 0; h < R / 4; ++h) {                            // samples 4h .. 4h+3 of the row
        SA[r][2 * h] = prmt(rows[r][2 * h], rows[r][2 * h + 1], 0x5410);          // (4h, 4h+2)
        SA[r][2 * h + 1] = prmt(rows[r][2 * h], rows[r][2 * h + 1], 0x7632);      // (4h+1, 4h+3)
      }
    // transposed: ST[r] = column r: pairs (A[c][r], A[c+2][r]) for c = 0, 1, 4, 5
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const uint32_t sel = (r & 1) ? 0x7632u : 0x5410u;
#pragma unroll
      for (int q = 0; q < R / 4; ++q) {
        ST[r][2 * q] = prmt(rows[4 * q + 0][r >> 1], rows[4 * q + 2][r >> 1], sel);
        ST[r][2 * q + 1] = prmt(rows[4 * q + 1][r >> 1], rows[4 * q + 3][r >> 1], sel);
      }
    }
  } else {
    uint32_t rows[R][K / 2 + (K < 2 ? 1 : 0)];                   // raw bytes: R rows of R bytes
    const int bx = valid ? blk % blocks_x : 0, by = valid ? blk / blocks_x : 0;
    const uint8_t *p = reinterpret_cast<const uint8_t *>(src) + (long)(by * W + sy * R) * stride + bx * W + sx * R;
#pragma unroll
    for (int r = 0; r < R; ++r) {
      if constexpr (R == 8) {
        const uint2 v = valid ? __ldg(reinterpret_cast<const uint2 *>(p + (long)r * stride)) : make_uint2(0, 0);
        rows[r][0] = v.x; rows[r][1] = v.y;
      } else {
        rows[r][0] = valid ? __ldg(reinterpret_cast<const uint32_t *>(p + (long)r * stride)) : 0u;
      }
    }
#pragma unroll
    for (int r = 0; r < R; ++r)
#pragma unroll
      for (int h = 0; h < R / 4; ++h) {
        SA[r][2 * h] = prmt(rows[r][h], 0u, 0x4240);
        SA[r][2 * h + 1] = prmt(rows[r][h], 0u, 0x4341);
      }
    // transposed: ST[r] holds column r of the block: pairs (A[c][r], A[c+2][r])
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const int h = r >> 2, b = r & 3;                            // byte b of word h in every row
#pragma unroll
      for (int q = 0; q < R / 4; ++q) {                           // q selects source rows 4q .. 4q+3
        const uint32_t sel = (uint32_t)b | ((uint32_t)(b + 4) << 4);
        const uint32_t t02 = prmt(rows[4 * q + 0][h], rows[4 * q + 2][h], sel);   // bytes: A[4q][r], A[4q+2][r]
        const uint32_t t13 = prmt(rows[4 * q + 1][h], rows[4 * q + 3][h], sel);
        ST[r][2 * q] = prmt(t02, 0u, 0x4140);
        ST[r][2 * q + 1] = prmt(t13, 0u, 0x4140);
      }
    }
  }

  for (int m = warp; m < 35; m += 4) {
    int d[R][K];
    if (m < 2) {
      // planar / DC: closed forms per sample (2 of 35 modes)
      const T *top = s_ref[g][m == 0 && LOG2W > 2 ? 2 : 0], *left = s_ref[g][m == 0 && LOG2W > 2 ? 3 : 1];
      const int dc = s_dc[g];
#pragma unroll
      for (int r = 0; r < R; ++r) {
#pragma unroll
        for (int k = 0; k < K; ++k) {
          const int c0 = (k >> 1) * 4 + (k & 1), y = sy * R + r;
          int v0, v1;
          if (m == 0) {
            v0 = planar_px(LOG2W, top, left, sx * R + c0, y);
            v1 = planar_px(LOG2W, top, left, sx * R + c0 + 2, y);
          } else if (LOG2W < 5) {
            v0 = filtered_dc_px(top, left, dc, sx * R + c0, y);
            v1 = filtered_dc_px(top, left, dc, sx * R + c0 + 2, y);
          } else {
            v0 = v1 = dc;
          }
          d[r][k] = (int)SA[r][k] - (v0 | (v1 << 16));
        }
      }
    } else {
      const bool vertical = m >= 18;
      const int mdisp = vertical ? m - 26 : 10 - m;
      const int adisp = abs(mdisp);
      const int sdisp = mdisp < 0 ? -ang_disp(adisp) : ang_disp(adisp);
      const int filt = intra_uses_filtered(LOG2W, m, 0) ? 2 : 0;
      const int main_sel = (vertical ? 0 : 1) + filt, side_sel = (vertical ? 1 : 0) + filt;
      const T *ext = s_plain[g][main_sel];
      if (sdisp < 0) {
        // main reference extended to negative indices by projecting the side reference (ref: intra-generic.c:88-108)
        const int inv = ang_inv(adisp);
        __syncwarp();
        for (int e = lane; e < GROUP * 2 * W; e += 32) {
          const int gb = e / (2 * W), j = e - gb * 2 * W, idx = j - W;
          s_ext[warp][gb][j] = idx >= -1 ? s_ref[gb][main_sel][idx + 1] : s_ref[gb][side_sel][min((128 + (-idx - 1) * inv) >> 8, 2 * W)];
        }
        __syncwarp();
        ext = s_ext[warp][g];
      }
      // sub-block position in the orientation being computed (transposed for horizontal modes)
      const int ex = vertical ? sx : sy, ey = vertical ? sy : sx;
      const bool edge = LOG2W < 5 && (m == 10 || m == 26) && ex == 0;         // ref: intra.c:293-300
      const T *side_unf = s_ref[g][vertical ? 1 : 0];
#pragma unroll
      for (int r = 0; r < R; ++r) {
        const int pos = (ey * R + r + 1) * sdisp;
        const int di = pos >> 5;
        const uint32_t f1 = (uint32_t)(pos & 31), f0 = 32u - f1;
        const int j0 = ex * R + di + W;
        uint32_t P[K];
        if constexpr (WIDE) {
          // words of two samples; an odd start index is a 16-bit funnel shift
          const uint32_t *wp = reinterpret_cast<const uint32_t *>(ext + (j0 & ~1));
          const uint32_t sh = (uint32_t)(j0 & 1) * 16;
          if constexpr (R == 8) {
            const uint32_t a0 = wp[0], a1 = wp[1], a2 = wp[2], a3 = wp[3], a4 = wp[4], a5 = sh ? wp[5] : 0u;
            const uint32_t w0 = __funnelshift_r(a0, a1, sh), w1 = __funnelshift_r(a1, a2, sh), w2 = __funnelshift_r(a2, a3, sh),
                           w3 = __funnelshift_r(a3, a4, sh), w4 = __funnelshift_r(a4, a5, sh);
            const uint32_t L0 = prmt(w0, w1, 0x5410), L1 = prmt(w0, w1, 0x7632), L2 = prmt(w1, w2, 0x5410);
            const uint32_t L4 = prmt(w2, w3, 0x5410), L5 = prmt(w2, w3, 0x7632), L6 = prmt(w3, w4, 0x5410);
            P[0] = interp2<T>(L0, L1, f0, f1); P[1] = interp2<T>(L1, L2, f0, f1);
            P[2] = interp2<T>(L4, L5, f0, f1); P[3] = interp2<T>(L5, L6, f0, f1);
          } else {
            const uint32_t a0 = wp[0], a1 = wp[1], a2 = wp[2], a3 = sh ? wp[3] : 0u;
            const uint32_t w0 = __funnelshift_r(a0, a1, sh), w1 = __funnelshift_r(a1, a2, sh), w2 = __funnelshift_r(a2, a3, sh);
            const uint32_t L0 = prmt(w0, w1, 0x5410), L1 = prmt(w0, w1, 0x7632), L2 = prmt(w1, w2, 0x5410);
            P[0] = interp2<T>(L0, L1, f0, f1); P[1] = interp2<T>(L1, L2, f0, f1);
          }
        } else {
        const uint32_t *wp = reinterpret_cast<const uint32_t *>(reinterpret_cast<const uint8_t *>(ext) + (j0 & ~3));
        const uint32_t sh = (uint32_t)(j0 & 3) * 8;
        if constexpr (R == 8) {
          const uint32_t a0 = wp[0], a1 = wp[1], a2 = wp[2];
          const uint32_t w0 = __funnelshift_r(a0, a1, sh), w1 = __funnelshift_r(a1, a2, sh), w2 = a2 >> sh;
          const uint32_t L0 = prmt(w0, 0u, 0x4240), L1 = prmt(w0, 0u, 0x4341), L4 = prmt(w1, 0u, 0x4240), L5 = prmt(w1, 0u, 0x4341);
          const uint32_t L2 = prmt(L0, L4, 0x5432), L6 = prmt(L4, w2, 0x1432);
          P[0] = interp2<T>(L0, L1, f0, f1); P[1] = interp2<T>(L1, L2, f0, f1);
          P[2] = interp2<T>(L4, L5, f0, f1); P[3] = interp2<T>(L5, L6, f0, f1);
        } else {
          const uint32_t a0 = wp[0], a1 = wp[1];
          const uint32_t w0 = __funnelshift_r(a0, a1, sh), w1 = a1 >> sh;
          const uint32_t L0 = prmt(w0, 0u, 0x4240), L1 = prmt(w0, 0u, 0x4341), L2 = prmt(L0, w1, 0x1432);
          P[0] = interp2<T>(L0, L1, f0, f1); P[1] = interp2<T>(L1, L2, f0, f1);
        }
        }
        if (edge) {   // first column: the edge filter of modes 10 / 26 (displacement 0)
          const int v = intra_edge_px<T>((int)(P[0] & 0xffffu), side_unf[ey * R + r + 1], side_unf[0]);
          P[0] = (P[0] & 0xffff0000u) | (uint32_t)v;
        }
#pragma unroll
        for (int k = 0; k < K; ++k) d[r][k] = (int)(vertical ? SA[r][k] : ST[r][k]) - (int)P[k];
      }
    }
    uint32_t cost;
    if constexpr (R == 8) cost = (hadamard8x8_lanes(d) + 2) >> 2;
    else cost = (hadamard4x4_lanes(d) + 1) >> 1;
#pragma unroll
    for (int o = SUBS / 2; o > 0; o >>= 1) cost += __shfl_xor_sync(0xffffffffu, cost, o);
    if (sub == 0) s_cost[g][m] = W >= 8 ? cost >> (PixTraits<T>::bd - 8) : cost;   // satd_NxN shifts by the extra bit depth, satd_4x4 does not
  }
  __syncthreads();
  // ---- the 35 costs of every block (optional) and the fused selection: first minimum (search order of the pass)
  if (costs)
    for (int e = threadIdx.x; e < GROUP * 35; e += 128) {
      const int gb = e / 35, m = e - gb * 35;
      if (first + gb < nblk) costs[(size_t)(first + gb) * 35 + m] = s_cost[gb][m];
    }
  if (best_mode && threadIdx.x < GROUP && first + (int)threadIdx.x < nblk) {
    uint32_t bc = s_cost[threadIdx.x][0];
    int bm = 0;
    for (int m = 1; m < 35; ++m) { const uint32_t c = s_cost[threadIdx.x][m]; if (c < bc) { bc = c; bm = m; } }
    best_mode[first + threadIdx.x] = (int8_t)bm;
    best_cost[first + threadIdx.x] = bc;
  }
}

template <class T, int LOG2W>
static int launch(const T *src, const T *rec, int stride, int pic_w, int pic_h, uint32_t *costs, int8_t *best_mode,
                  uint32_t *best_cost, cudaStream_t st)
{
  constexpr int W = 1 << LOG2W, SUBS = W >= 8 ? (W / 8) * (W / 8) : 1, GROUP = 32 / SUBS;
  const int bx = pic_w / W, nblk = bx * (pic_h / W);
  if (nblk == 0) return 0;
  rough_search_u8_kernel<T, LOG2W><<<(nblk + GROUP - 1) / GROUP, 128, 0, st>>>(src, rec, stride, pic_w, pic_h, bx, nblk, costs, best_mode, best_cost);
  KVZC_LAUNCHED();
  return 0;
}

// costs (35 per block) and best_mode/best_cost (one per block) are both optional outputs
int rough_search_u8(int log2w, const uint8_t *src, const uint8_t *rec, int stride, int pic_w, int pic_h, uint32_t *costs,
                    int8_t *best_mode, uint32_t *best_cost, cudaStream_t st)
{
  switch (log2w) {
    case 2: return launch<uint8_t, 2>(src, rec, stride, pic_w, pic_h, costs, best_mode, best_cost, st);
    case 3: return launch<uint8_t, 3>(src, rec, stride, pic_w, pic_h, costs, best_mode, best_cost, st);
    case 4: return launch<uint8_t, 4>(src, rec, stride, pic_w, pic_h, costs, best_mode, best_cost, st);
    default: return launch<uint8_t, 5>(src, rec, stride, pic_w, pic_h, costs, best_mode, best_cost, st);
  }
}

// the same for 16-bit samples (10-bit video)
int rough_search_u16(int log2w, const uint16_t *src, const uint16_t *rec, int stride, int pic_w, int pic_h, uint32_t *costs,
                     int8_t *best_mode, uint32_t *best_cost, cudaStream_t st)
{
  switch (log2w) {
    case 2: return launch<uint16_t, 2>(src, rec, stride, pic_w, pic_h, costs, best_mode, best_cost, st);
    case 3: return launch<uint16_t, 3>(src, rec, stride, pic_w, pic_h, costs, best_mode, best_cost, st);
    case 4: return launch<uint16_t, 4>(src, rec, stride, pic_w, pic_h, costs, best_mode, best_cost, st);
    default: return launch<uint16_t, 5>(src, rec, stride, pic_w, pic_h, costs, best_mode, best_cost, st);
  }
}

}  // namespace kvzc
