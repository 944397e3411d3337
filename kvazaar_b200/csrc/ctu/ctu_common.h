// ctu_common.h -- types, tables and the execution model of the device-resident CTU search driver (SURVEY §8f rank 2).
//
// ONE source, two compilations:
//   * nvcc, sm_90a: the product.  One CTA (four warps) owns one CTU at a time; every function is called by ALL threads
//     of the CTA with uniform control flow unless it takes a Team (ctu_leaf.h): then the CTA's warps run independent
//     transform-unit jobs side by side and synchronise inside their warp only.  Scalar decisions live in a
//     shared-memory state block that only the leader (lane 0 of one warp) mutates between barriers -- and every thread
//     copies the state it branches on BEFORE the barrier after which the leader may change it; data-parallel phases
//     are item-strided loops over the CTA.
//   * g++ (tests/hostsim, TEST INFRASTRUCTURE): the same code with a CTA of one thread and no-op barriers, so the
//     control flow can be debugged against the compiled reference on a machine without a GPU.  The product
//     never runs this build.
#pragma once
#include <stdint.h>
#include <stddef.h>
#include <string.h>
#include "../coeff_rules.h"
#include "../pixel_rules.h"

#if defined(__CUDACC__)
#define CTU_FN __device__ __forceinline__
#define CTU_FN_NOINLINE __device__ __noinline__
#define CTU_MFN __device__ __forceinline__
#else
#define CTU_FN static inline
#define CTU_FN_NOINLINE static
#define CTU_MFN inline
#endif

#if defined(__CUDA_ARCH__)
#define CTU_TID ((int)threadIdx.x)
#define CTU_NT ((int)blockDim.x)
#define CTU_SYNC() __syncthreads()
// the algorithms with a serial spine (RDOQ) run on at most one warp of a team, so that their inner synchronisation is a
// warp barrier; the rest of the CTA waits at the next CTA barrier
#define CTU_TEAM_N 32
#else
#define CTU_TID 0
#define CTU_NT 1
#define CTU_SYNC() ((void)0)
#define CTU_TEAM_N 1
#endif
// The leader is lane 0 of ONE of the CTA's warps, chosen per CTA (first word of the CTA's shared memory, set by the kernel):
// the CTAs that share an SM get different leader warps, so their serial sections run on different SM sub-partitions
// (own scheduler, own L0 instruction cache) instead of all on warp 0's.
#if defined(__CUDACC__)
extern __shared__ __align__(16) unsigned char ctu_smem_raw[];
#endif
#if defined(__CUDA_ARCH__)
#define CTU_LEADER_TID (*reinterpret_cast<const int *>(ctu_smem_raw))
#else
#define CTU_LEADER_TID 0
#endif
#define CTU_LEADER if (CTU_TID == CTU_LEADER_TID)

// Shared-window addressing.  Inside a __noinline__ function ptxas cannot see where a pointer argument points, so loads
// and stores through it are generic (LD / ST: the L1TEX path and its long scoreboard) even when every caller passes
// shared memory.  sm(p) re-derives such a pointer from the shared-memory symbol: accesses through the result compile to
// LDS / STS, and it costs one or two integer operations.  Only for objects that are ALWAYS in the CTA's shared memory
// (CtuST and what is carved out of it); the identity in the host build.  The offset is taken with cvta (the shared
// address of p), not as the difference of two generic pointers: with that form the search spine's build faulted on
// the device although every pointer it was given lay inside the window.
#if defined(__CUDA_ARCH__)
template <typename T> CTU_FN T *sm(T *p)
{
  const unsigned off = (unsigned)__cvta_generic_to_shared(p) - (unsigned)__cvta_generic_to_shared(ctu_smem_raw);
  return reinterpret_cast<T *>(ctu_smem_raw + off);
}
#else
template <typename T> CTU_FN T *sm(T *p) { return p; }
#endif

// Frame-level data (reconstruction planes, CU records, border buffers, SAO parameters, row context models) is written
// by the CTA of one CTU and read by the CTAs of its neighbours, which run on other SMs inside the same launch: such
// loads must be served by L2 (ld.global.cg), never by a possibly stale line of this SM's L1.
#if defined(__CUDA_ARCH__)
#define CTU_LD_FRAME(p) __ldcg(p)
#else
#define CTU_LD_FRAME(p) (*(p))
#endif

// Phase profile (diagnostic build, make PROF=1): cycles of the leader thread per phase, summed over all CTUs.
// PR_QRES4 .. PR_QRES32: transform-unit job batches whose largest unit is 4x4, 8x8, 16x16, 32x32 (pr_qres_of).
// PR_COEFFCOST: the coefficient bits of the RDO candidates' jobs that ran on the leader's team (a part of their batch's
// time).
enum { PR_LOAD, PR_SEARCH, PR_STORE, PR_DEBLOCK, PR_SAO, PR_TRACK, PR_REFS, PR_SATD, PR_REPLAY, PR_QRES4, PR_QRES8, PR_QRES16, PR_QRES32,
       PR_COST, PR_COPY, PR_COEFFCOST, PR_WAIT, PR_CHROMA, PR_RDO_LOOP, PR_WRITEBACK, PR_N };
#define pr_qres_of(log2n) (PR_QRES4 + (log2n) - 2)
#if defined(KVZ_CTU_PROF) && defined(__CUDA_ARCH__)
#define PROF_T0(id) const long long prof_t0_##id = clock64()
#define PROF_ADD(S, id) do { if (CTU_TID == CTU_LEADER_TID) (S)->prof[id] += clock64() - prof_t0_##id; } while (0)
#define PROF_ADD_AS(S, id, as) do { if (CTU_TID == CTU_LEADER_TID) (S)->prof[as] += clock64() - prof_t0_##id; } while (0)
#else
#define PROF_T0(id) ((void)0)
#define PROF_ADD(S, id) ((void)0)
#define PROF_ADD_AS(S, id, as) ((void)0)
#endif

namespace kvzctu {

using namespace kvzcoeff;
// The algorithm is compiled once per sample type (PixTraits): uint8_t for 8-bit, uint16_t for 10-bit pictures.
using namespace kvzpix;

// ---------------------------------------------------------------------------------------------- configuration
// Mirrors the fields of kvz_config / encoder_control_t / encoder_state_t the intra CTU search reads
// (ref: src/search.c:646-1068, src/search_intra.c, src/intra.c, src/transform.c, src/rdo.c, src/sao.c, src/filter.c).
struct CtuConfig {
  int32_t width, height;            // luma samples, multiples of 8 (cfg.width/height after padding)
  int32_t qp;                       // state->qp == state->frame->QP (fixed QP, no rate control)
  int32_t rdo;                      // cfg.rdo 0..3
  int32_t pu_depth_intra_min, pu_depth_intra_max;   // cfg.pu_depth_intra.{min,max}[0]
  int32_t rdoq_enable, rdoq_skip, signhide_enable, trskip_enable;
  int32_t sao_type;                 // cfg.sao_type: 0 off, 1 edge, 2 band, 3 full
  int32_t deblock_enable, deblock_beta, deblock_tc;
  int32_t cu_split_termination;     // 0 = zero (KVZ_CU_SPLIT_TERMINATION_ZERO), 1 = off
  int32_t intra_rdo_et, combine_intra_cus, intra_chroma_search, full_intra_search;
  int32_t wpp;
  int32_t bitdepth;                 // 0 or 8: 8-bit samples, 10: 10-bit samples
  double lambda, lambda_sqrt;       // state->lambda, state->lambda_sqrt
};

// ---------------------------------------------------------------------------------------------- CU records
// The fields of cu_info_t (ref: src/cu.h:126-165) an intra CU uses, unpacked.
struct alignas(4) CuRec {
  uint8_t type, depth, part_size, tr_depth;
  uint8_t tr_skip, qp;
  int8_t mode, mode_chroma;
  uint16_t cbf;
  uint16_t pad;
};
static_assert(sizeof(CuRec) == 12, "CuRec layout");
CTU_FN CuRec ld_frame_cu(const CuRec *p)
{
  union { CuRec c; uint32_t w[3]; } u;
  const uint32_t *q = (const uint32_t *)p;
  u.w[0] = CTU_LD_FRAME(q); u.w[1] = CTU_LD_FRAME(q + 1); u.w[2] = CTU_LD_FRAME(q + 2);
  return u.c;
}
enum { CU_NOTSET = 0, CU_INTRA = 1 };
enum { SIZE_2Nx2N = 0, SIZE_NxN = 3 };
enum { COLOR_Y = 0, COLOR_U = 1, COLOR_V = 2 };

// cbf helpers (ref: src/cu.h:505-566)
CTU_FN uint16_t cbf_mask(int depth) { return (uint16_t)(0x1f >> depth); }
CTU_FN int cbf_is_set(uint16_t cbf, int depth, int plane) { return (cbf & (cbf_mask(depth) << (5 * plane))) != 0; }
CTU_FN int cbf_is_set_any(uint16_t cbf, int depth) { return cbf_is_set(cbf, depth, 0) || cbf_is_set(cbf, depth, 1) || cbf_is_set(cbf, depth, 2); }
CTU_FN void cbf_set(uint16_t *cbf, int depth, int plane) { *cbf |= (uint16_t)((0x10 >> depth) << (5 * plane)); }
CTU_FN void cbf_clear(uint16_t *cbf, int depth, int plane) { *cbf &= (uint16_t)~(cbf_mask(depth) << (5 * plane)); }
CTU_FN void cbf_copy(uint16_t *cbf, uint16_t src, int plane) { cbf_clear(cbf, 0, plane); *cbf |= (uint16_t)(src & (0x1f << (5 * plane))); }
CTU_FN void cbf_set_conditionally(uint16_t *cbf, const uint16_t child[3], int depth, int plane)
{
  if (cbf_is_set(child[0], depth + 1, plane) || cbf_is_set(child[1], depth + 1, plane) || cbf_is_set(child[2], depth + 1, plane)) cbf_set(cbf, depth, plane);
}

// One level of the work tree (ref: lcu_t, src/cu.h:299-337, and work_tree[], src/search.c:1220-1224).  The CU records
// are what the serial decision code reads all the time: they live in shared memory (CtuS); the pixel and coefficient
// planes of the level stay in global memory (LcuStore) and are only touched by data-parallel phases.  The source pixels
// and the border references are the same on every level and live in CtuWork.
template <typename Pix> struct LcuStore {
  Pix rec_y[64 * 64], rec_u[32 * 32], rec_v[32 * 32];
  int16_t coeff_y[64 * 64], coeff_u[32 * 32], coeff_v[32 * 32];
};
template <typename Pix> struct LcuLevel {
  CuRec cu[17 * 17 + 1];
  Pix *rec_y, *rec_u, *rec_v;
  int16_t *coeff_y, *coeff_u, *coeff_v;
};
template <typename Pix> CTU_FN CuRec *cu_at(LcuLevel<Pix> *L, int x_px, int y_px) { return &L->cu[18 + (x_px >> 2) + (y_px >> 2) * 17]; }   // LCU_GET_CU_AT_PX
template <typename Pix> CTU_FN CuRec *cu_top_right(LcuLevel<Pix> *L) { return &L->cu[17 * 17]; }

// z-order offset of a 4-aligned position inside a plane of `width` (ref: xy_to_zorder, src/cu.h:367-402)
CTU_FN int zorder(int width, int x, int y)
{
  int r = 0;
  if (width == 64) { r += (x >> 5) * 1024 + (y >> 5) * 2048; x &= 31; y &= 31; }
  if (width >= 32) { r += (x >> 4) * 256 + (y >> 4) * 512; x &= 15; y &= 15; }
  if (width >= 16) { r += (x >> 3) * 64 + (y >> 3) * 128; x &= 7; y &= 7; }
  if (width >= 8) { r += (x >> 2) * 16 + (y >> 2) * 32; }
  return r;
}

// ---------------------------------------------------------------------------------------------- CABAC models
// The models as a memory image of cabac_data_t.ctx (offsets: CtxOff, coeff_rules.h).
struct alignas(16) CabacState {     // 192 bytes: copied around every speculative branch, as 16-byte moves
  uint8_t ctx[CTX_COUNT];
  uint8_t update;          // cabac_data_t.update travels with every copy of the struct (ref: search.c:655, 956-958)
  uint8_t pad[7];
};

// ---------------------------------------------------------------------------------------------- SAO
struct SaoRec {            // sao_info_t (ref: src/sao.h)
  int32_t type;            // 0 none, 1 band, 2 edge
  int32_t eo_class;
  int32_t ddistortion;
  int32_t merge_left_flag, merge_up_flag;
  int32_t band_position[2];
  int32_t offsets[10];
};

// ---------------------------------------------------------------------------------------------- tables
struct CtuTables {
  uint16_t scan[3][4][1024];        // [scan_idx][log2n - 2][scan position] -> raster position (kvz_g_sig_last_scan)
  uint8_t scan_cg[3][4][64];        // [scan_idx][log2n - 2][i] -> coefficient group (raster) of scan group i
  uint8_t ref_top[16][16];          // number of available reference pixels above / left by 4x4 position in the LCU
  uint8_t ref_left[16][16];         //   (ref: src/intra.c:47-82: what the z-order coding order has reconstructed)
  int8_t tr[4][32 * 32];            // DCT matrices M[k][i] for n = 4, 8, 16, 32 (ref: dct-generic.c:38-120)
  int8_t dst4[16];
  int32_t ebits[128];               // kvz_entropy_bits (ref: rdo.c:69-79): [state byte ^ bin], 15 fractional bits
  uint8_t next_mps[128], next_lps[128];   // kvz_g_auc_next_state_* (ref: cabac.c:40-62)
  uint8_t sig_ctx4[16];             // ctx_ind_map of 4x4 blocks (ref: context.c:366)
  uint8_t group_idx[32], min_in_group[10];
};

// ---- host-side table construction (product host code and the test build share it)
inline void ctu_tables_init(CtuTables *t)
{
  memset(t, 0, sizeof(*t));
  for (int s = 0; s < 3; ++s)
    for (int l = 2; l <= 5; ++l) {
      const int n = 1 << l, gw = n >> 2;
      // the reference only has horizontal / vertical tables up to 8x8; larger blocks always scan diagonally
      for (int i = 0; i < n * n; ++i) {
        int pos;
        if (l == 2) pos = scan_small(s, 2, i);
        else {
          const int cg = scan_small(l >= 4 ? 0 : s, l - 2, i >> 4), in = scan_small(l >= 4 ? 0 : s, 2, i & 15);
          pos = ((cg / gw) * 4 + (in >> 2)) * n + (cg % gw) * 4 + (in & 3);
        }
        t->scan[s][l - 2][i] = (uint16_t)pos;
      }
      for (int i = 0; i < gw * gw; ++i) {
        const int first = t->scan[s][l - 2][i << 4];
        t->scan_cg[s][l - 2][i] = (uint8_t)(((first >> l) >> 2) * gw + ((first & (n - 1)) >> 2));
      }
    }
  for (int uy = 0; uy < 16; ++uy)
    for (int ux = 0; ux < 16; ++ux) {
      t->ref_top[uy][ux] = (uint8_t)ref_px_top(uy, ux);
      t->ref_left[uy][ux] = (uint8_t)ref_px_left(uy, ux);
    }
  static const int8_t c32[33] = { 64, 90, 90, 90, 89, 88, 87, 85, 83, 82, 80, 78, 75, 73, 70, 67, 64,
                                  61, 57, 54, 50, 46, 43, 38, 36, 31, 25, 22, 18, 13, 9, 4, 0 };
  for (int l = 2; l <= 5; ++l) {
    const int n = 1 << l;
    for (int k = 0; k < n; ++k)
      for (int i = 0; i < n; ++i) {
        int m = ((k * (32 / n)) * (2 * i + 1)) & 127;
        if (m > 64) m = 128 - m;
        t->tr[l - 2][k * n + i] = (int8_t)(m <= 32 ? c32[m] : -c32[64 - m]);
      }
  }
  static const int8_t dst[16] = { 29, 55, 74, 84, 74, 74, 0, -74, 84, -29, -74, 55, 55, -84, 74, -29 };
  memcpy(t->dst4, dst, 16);
  static const int32_t mps[64] = { COEFF_EBITS_MPS }, lps[64] = { COEFF_EBITS_LPS };
  for (int i = 0; i < 128; ++i) t->ebits[i] = (i & 1) ? lps[i >> 1] : mps[i >> 1];
  for (int uc = 0; uc < 128; ++uc) {
    t->next_mps[uc] = cabac_next_mps(uc);
    t->next_lps[uc] = cabac_next_lps(uc);
  }
  static const uint8_t map4[16] = { COEFF_SIG_CTX4 };
  memcpy(t->sig_ctx4, map4, 16);
  for (int x = 0; x < 32; ++x) t->group_idx[x] = (uint8_t)last_group(x);
  static const uint8_t mig[10] = { COEFF_MIN_IN_GROUP };
  memcpy(t->min_in_group, mig, 10);
}

// kvz_get_scan_order (ref: src/encoderstate.c:1761-1775), CU_INTRA only
CTU_FN int scan_order_intra(int mode, int depth)
{
  if (depth >= 3) {
    if (mode >= 6 && mode <= 14) return 2;    // SCAN_VER
    if (mode >= 22 && mode <= 30) return 1;   // SCAN_HOR
  }
  return 0;
}

// kvz_get_scaled_qp with the qp_offset of the bit depth, 6 * (bd - 8) (ref: quant-generic.c:57, 305; rdo.c:672); the
// search's QP is never negative, so the offset can be added after the chroma mapping
template <typename Pix> CTU_FN int scaled_qp_px(int type, int qp) { return scaled_qp(type, qp, 0) + 6 * (PixTraits<Pix>::bd - 8); }

}  // namespace kvzctu
