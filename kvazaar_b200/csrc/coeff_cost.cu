// coeff_cost.cu -- CABAC bit cost of the quantised coefficients of a TU (SURVEY §8f rank 1: "coefficient bit-cost
// estimation"): what kvz_get_coeff_cost's CABAC branch computes (src/rdo.c:223-264, 291-330) by running
// kvz_encode_coeff_nxn in only_count mode (src/strategies/generic/encode_coding_tree-generic.c:40-290) together with
// kvz_encode_last_significant_xy (src/encode_coding_tree.c:63-115) and kvz_cabac_write_coeff_remain (src/cabac.c:275-301).
//
// The count itself is coeff_bits (coeff_rules.h), in units of 2^-15 bit.  With `update` the context models adapt
// inside the TU exactly as CABAC_BIN would; every TU of a batch starts from the same context image.  One thread per TU,
// or (16x16 and 32x32 grids, no adaptation) one warp per TU.
#include "rdoq.cuh"

namespace kvzc {

// coeff_bits' policy: scans computed, entropy bits staged in shared memory (rdoq_load_ebits), the models of this TU
struct CostWalk {
  uint8_t *models;            // this TU's (possibly private) context image
  const int32_t *eb;
  bool update, trskip, sh;
  int32_t abs_coeff[16];
  struct Scan { int scan_idx, log2n; __device__ int operator[](int i) const { return scan_pos(scan_idx, log2n, i); } };
  struct ScanCg {
    int scan_idx, log2n;
    __device__ int operator[](int i) const
    {
      const int first = scan_pos(scan_idx, log2n, i << 4), n = 1 << log2n;
      return ((first >> log2n) >> 2) * (n >> 2) + ((first & (n - 1)) >> 2);
    }
  };
  __device__ Scan scan(int scan_idx, int log2n) const { return Scan{ scan_idx, log2n }; }
  __device__ ScanCg scan_cg(int scan_idx, int log2n) const { return ScanCg{ scan_idx, log2n }; }
  __device__ int group_idx(int x) const { return last_group(x); }
  __device__ SigCtx4 sig_ctx4() const { return SigCtx4(); }
  __device__ int32_t *abs_scratch() { return abs_coeff; }
  __device__ bool trskip_enable() const { return trskip; }
  __device__ bool signhide() const { return sh; }
  __device__ void bin(int off, int val, long long *bits)
  {
    const uint8_t st = models[off];
    *bits += eb[st ^ val];
    if (update) models[off] = ((st & 1) == val) ? cabac_next_mps(st) : cabac_next_lps(st);
  }
};

__global__ void __launch_bounds__(128) coeff_cost_kernel(kvz_cuda_coeff_cost_params p, const kvz_cuda_cabac_ctx *__restrict__ cabac,
                                                         const int16_t *__restrict__ coeff, int n, const kvz_cuda_rdoq_tu *__restrict__ tus,
                                                         int count, double *__restrict__ bits_out, kvz_cuda_cabac_ctx *__restrict__ ctx_out)
{
  __shared__ kvz_cuda_cabac_ctx s_ctx;
  __shared__ int32_t s_ebits[128];
  rdoq_load_ebits(s_ebits);
  for (int i = threadIdx.x; i < (int)sizeof(kvz_cuda_cabac_ctx); i += blockDim.x) ((uint8_t *)&s_ctx)[i] = ((const uint8_t *)cabac)[i];
  __syncthreads();
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= count) return;
  const kvz_cuda_rdoq_tu tu = tus[t];
  kvz_cuda_cabac_ctx mine;                       // private copy only when the models adapt
  CostWalk c;
  c.eb = s_ebits; c.update = p.update != 0; c.trskip = p.trskip_enable != 0; c.sh = p.signhide_enable != 0;
  if (c.update) { mine = s_ctx; c.models = (uint8_t *)&mine; } else c.models = (uint8_t *)&s_ctx;
  const int log2n = 31 - __clz(n);
  const long long bits = coeff_bits(c, coeff + tu.off_coef, log2n, tu.type, tu.scan_idx, tu.block_type /* tr_skip flag */, COEFF_NO_MASK);
  bits_out[t] = (double)bits * (1.0 / 32768.0);
  if (c.update && ctx_out) ctx_out[t] = mine;
}

// Uniform TU grid of the frame-level pass (TU t at coeff[t * n * n], intra; scan from the intra mode as in the
// reconstruction kernel).  No context adaptation; transform skip disabled.
__global__ void __launch_bounds__(128) coeff_cost_grid_kernel(int signhide, int trskip_enable, const kvz_cuda_cabac_ctx *__restrict__ cabac,
                                                              const int16_t *__restrict__ coeff, const int16_t *__restrict__ coeff2, int count,
                                                              int log2n, const int8_t *__restrict__ modes, int is_chroma,
                                                              double *__restrict__ bits_out, double *__restrict__ bits_out2)
{
  __shared__ kvz_cuda_cabac_ctx s_ctx;
  __shared__ int32_t s_ebits[128];
  rdoq_load_ebits(s_ebits);
  for (int i = threadIdx.x; i < (int)sizeof(kvz_cuda_cabac_ctx); i += blockDim.x) ((uint8_t *)&s_ctx)[i] = ((const uint8_t *)cabac)[i];
  __syncthreads();
  int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (coeff2 ? 2 * count : count)) return;
  if (t >= count) { t -= count; coeff = coeff2; bits_out = bits_out2; }      // second plane (V) of a U+V launch
  const int w = 1 << log2n;
  int scan = 0;
  if ((!is_chroma && w <= 8) || (is_chroma && w == 4)) { const int m = modes[t]; scan = (m >= 6 && m <= 14) ? 2 : ((m >= 22 && m <= 30) ? 1 : 0); }
  CostWalk c;
  c.eb = s_ebits; c.update = false; c.trskip = trskip_enable != 0; c.sh = signhide != 0; c.models = (uint8_t *)&s_ctx;
  const long long bits = coeff_bits(c, coeff + (size_t)t * w * w, log2n, is_chroma ? 2 : 0, scan, 0, COEFF_NO_MASK);   // the flag is counted as 0 (rdo.c:251-258)
  bits_out[t] = (double)bits * (1.0 / 32768.0);
}


// ---- warp per TU, no context adaptation (16x16 and 32x32 grids) -------------------------------------------------------
// The count is exact in units of 2^-15 bit (coeff_bits), so the total does not depend on the order of the additions.
// Without adaptation that makes it position-parallel:
//   * a lane owns coefficient groups (scan index i = lane, lane + 32): non-zero mask, coefficient magnitudes in coding
//     order, whether one of its first eight magnitudes exceeds 1 (the only state a group hands to the next one:
//     "c1 == 0" selects the next group's context set);
//   * significance / coded-sub-block flags cost depends on static neighbour flags only;
//   * greater1 / greater2 / remaining-level bins are a short serial chain inside one group.
__device__ long long coeff_cost_tu_warp(const uint8_t *models, const int32_t *eb, const int16_t *__restrict__ coeff, int log2n, int type,
                                        int signhide, int lane, uint32_t *s_nz /* [64] shared: per-group masks by scan index */,
                                        uint8_t *s_raster /* [64] shared: group non-empty, by raster position */)
{
  const int n = 1 << log2n, side = n >> 2, ncg = side * side;
  auto cost = [&](int model_off, int val) { return (long long)eb[models[model_off] ^ val]; };
  CostWalk w;
  w.models = (uint8_t *)models; w.eb = eb; w.update = false;
  // pass 1: per group (scan order, diagonal: scan_idx is 0 for these sizes) the non-zero mask in coding order
  int my_abs[2][16];
  unsigned my_mask[2] = { 0, 0 };
  int my_blk[2] = { 0, 0 };
  for (int r = 0; r < 2; ++r) {
    const int i = lane + 32 * r;
    if (i >= ncg) break;
    const int first = scan_pos(0, log2n, i << 4);
    my_blk[r] = ((first >> log2n) >> 2) * side + ((first & (n - 1)) >> 2);
    const int by = (first >> log2n) & ~3, bx = (first & (n - 1)) & ~3;
#pragma unroll
    for (int k = 0; k < 16; ++k) {
      const int in = scan_small(0, 2, k);                             // position inside the 4x4 group
      const int v = coeff[(by + (in >> 2)) * n + bx + (in & 3)];
      my_abs[r][k] = abs(v);
      if (v) my_mask[r] |= 1u << k;
    }
    // bit 16: one of the group's first eight magnitudes in coding order (highest scan position first) exceeds 1
    unsigned gt1 = 0;
    for (int k = 15, seen = 0; k >= 0 && seen < 8; --k)
      if ((my_mask[r] >> k) & 1) { gt1 |= my_abs[r][k] > 1; ++seen; }
    s_nz[i] = my_mask[r] | (gt1 << 16);
    s_raster[my_blk[r]] = my_mask[r] != 0;
  }
  __syncwarp();
  // last group / last position
  int cg_last = -1;
  for (int r = 0; r < 2; ++r) if (my_mask[r]) cg_last = lane + 32 * r;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) cg_last = max(cg_last, __shfl_xor_sync(0xffffffffu, cg_last, o));
  if (cg_last < 0) return 0;
  const unsigned last_mask = s_nz[cg_last] & 0xffffu;
  const int k_last = 31 - __clz(last_mask), scan_last = cg_last * 16 + k_last;
  // s_raster: sig_coeffgroup_flag before the forced entries, by raster position
  auto flag_at = [&](int cgx, int cgy) { return s_raster[cgy * side + cgx] != 0; };
  long long sum = 0;
  if (lane == 0) {
    const int pos_last = scan_pos(0, log2n, scan_last);
    sum += last_pos_bits(w, pos_last & (n - 1), pos_last >> log2n, n, log2n, type);
  }
  const int base_cg = CTX_SIG_CG + type;
  const int base_sig = type == 0 ? CTX_SIG_LUMA : CTX_SIG_CHROMA;
  for (int r = 0; r < 2; ++r) {
    const int i = lane + 32 * r;
    if (i >= ncg || i > cg_last) continue;
    const unsigned mask = my_mask[r];
    const int cgy = my_blk[r] / side, cgx = my_blk[r] - cgy * side;
    const int right = (cgx < side - 1) ? (int)flag_at(cgx + 1, cgy) : 0;
    const int lower = (cgy < side - 1) ? (int)flag_at(cgx, cgy + 1) : 0;
    const bool coded = mask != 0 || i == 0;                               // forced for the first group; the last one is non-empty
    if (i != cg_last && i != 0) sum += cost(base_cg + (right || lower), mask != 0);
    if (!coded) continue;
    // sig_coeff_flag bins: every position below the last coefficient, except the group's first scan position when the
    // rest of the group was empty and the group is not the DC group (it is then inferred)
    const int pattern = right + (lower << 1);
    const int top = (i == cg_last) ? k_last - 1 : 15;
    const int first = scan_pos(0, log2n, i << 4);
    const int by = (first >> log2n) & ~3, bx = (first & (n - 1)) & ~3;
    for (int k = top; k >= 0; --k) {
      const bool earlier_nz = (mask >> (k + 1)) != 0;                      // a non-zero coefficient coded before this one in the group
      if (k > 0 || i == 0 || earlier_nz) {
        const int in = scan_small(0, 2, k);
        sum += cost(base_sig + sig_ctx_inc(SigCtx4(), pattern, 0, bx + (in & 3), by + (in >> 2), log2n, type), (mask >> k) & 1);
      }
    }
    if (!mask) continue;
    // level bins of the group's non-zero coefficients in coding order (highest scan position first)
    int abs_c[16], num_nz = 0;
    for (int k = 15; k >= 0; --k) if ((mask >> k) & 1) abs_c[num_nz++] = my_abs[r][k];
    const int last_nz = 31 - __clz(mask), first_nz = __ffs(mask) - 1;
    // context set: +1 when the previous coded group left c1 == 0, i.e. one of its first eight magnitudes exceeded 1
    int ctx_set = (i > 0 && type == 0) ? 2 : 0;
    for (int j = i + 1; j <= cg_last; ++j) {
      const unsigned pm = s_nz[j];
      if (!(pm & 0xffffu)) continue;
      ctx_set += (pm >> 16) & 1;
      break;
    }
    int c1 = 1, first_c2 = -1;
    const int base_one = (type == 0 ? CTX_ONE_LUMA : CTX_ONE_CHROMA) + 4 * ctx_set;
    const int num_c1 = min(num_nz, 8);
    for (int k = 0; k < num_c1; ++k) {
      const int symbol = abs_c[k] > 1;
      sum += cost(base_one + c1, symbol);
      if (symbol) { c1 = 0; if (first_c2 == -1) first_c2 = k; }
      else if (c1 < 3 && c1 > 0) ++c1;
    }
    if (c1 == 0 && first_c2 != -1) sum += cost((type == 0 ? CTX_ABS_LUMA : CTX_ABS_CHROMA) + ctx_set, abs_c[first_c2] > 2);
    sum += 32768ll * ((signhide && last_nz - first_nz >= 4) ? num_nz - 1 : num_nz);
    if (c1 == 0 || num_nz > 8) {
      int first_coeff2 = 1, rice = 0;
      for (int k = 0; k < num_nz; ++k) {
        const int base_level = (k < 8) ? (2 + first_coeff2) : 1;
        if (abs_c[k] >= base_level) {
          sum += 32768ll * coeff_remain_bits(abs_c[k] - base_level, rice);
          if (abs_c[k] > 3 * (1 << rice)) rice = min(rice + 1, 4);
        }
        if (abs_c[k] >= 2) first_coeff2 = 0;
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  return sum;
}

__global__ void __launch_bounds__(128) coeff_cost_grid_warp_kernel(int signhide, const kvz_cuda_cabac_ctx *__restrict__ cabac,
                                                                   const int16_t *__restrict__ coeff, const int16_t *__restrict__ coeff2, int count,
                                                                   int log2n, int is_chroma, double *__restrict__ bits_out, double *__restrict__ bits_out2)
{
  __shared__ kvz_cuda_cabac_ctx s_ctx;
  __shared__ int32_t s_ebits[128];
  __shared__ uint32_t s_nz[4][64];
  __shared__ uint8_t s_raster[4][64];
  rdoq_load_ebits(s_ebits);
  for (int i = threadIdx.x; i < (int)sizeof(kvz_cuda_cabac_ctx); i += blockDim.x) ((uint8_t *)&s_ctx)[i] = ((const uint8_t *)cabac)[i];
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int t = blockIdx.x * 4 + warp;
  if (t >= (coeff2 ? 2 * count : count)) return;
  if (t >= count) { t -= count; coeff = coeff2; bits_out = bits_out2; }
  const long long sum = coeff_cost_tu_warp((const uint8_t *)&s_ctx, s_ebits, coeff + ((size_t)t << (2 * log2n)), log2n, is_chroma ? 2 : 0, signhide, lane, s_nz[warp], s_raster[warp]);
  if (lane == 0) bits_out[t] = (double)sum * (1.0 / 32768.0);
}

int coeff_cost_launch_grid(int signhide, const kvz_cuda_cabac_ctx *ctx_dev, const int16_t *coeff, const int16_t *coeff2, int count, int log2n,
                           const int8_t *modes, int trskip_enable, double *bits_out, double *bits_out2, cudaStream_t st, int is_chroma)
{
  const int total = coeff2 ? 2 * count : count;
  if (log2n >= 4)      // 16x16 / 32x32: diagonal scan only, a warp per TU
    coeff_cost_grid_warp_kernel<<<(total + 3) / 4, 128, 0, st>>>(signhide, ctx_dev, coeff, coeff2, count, log2n, is_chroma, bits_out, bits_out2);
  else
    coeff_cost_grid_kernel<<<(total + 127) / 128, 128, 0, st>>>(signhide, trskip_enable, ctx_dev, coeff, coeff2, count, log2n, modes, is_chroma, bits_out, bits_out2);
  KVZC_LAUNCHED();
  return 0;
}

}  // namespace kvzc

using namespace kvzc;

extern "C" int kvz_cuda_coeff_cost_batch(const kvz_cuda_coeff_cost_params *p, const kvz_cuda_cabac_ctx *ctx_dev, const int16_t *coeff, int n,
                                         const kvz_cuda_rdoq_tu *tus, int count, double *bits_out, kvz_cuda_cabac_ctx *ctx_out, void *stream)
{
  KVZC_REQUIRE_DEVICE();
  KVZC_ARG(p && ctx_dev && coeff && tus && bits_out && count >= 0);
  KVZC_ARG(n == 4 || n == 8 || n == 16 || n == 32);
  if (count == 0) return 0;
  coeff_cost_kernel<<<(count + 127) / 128, 128, 0, as_stream(stream)>>>(*p, ctx_dev, coeff, n, tus, count, bits_out, ctx_out);
  KVZC_LAUNCHED();
  return 0;
}
