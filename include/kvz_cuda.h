/*
 * kvz_cuda.h -- C ABI of libkvzcuda.so: an H100 (sm_90a) "cuda" strategy for Kvazaar's
 * per-CTU strategy kernels (reference: Kvazaar's src/strategies, SURVEY.md section 8).
 *
 * Plain C, no reference headers, no torch types: pointers, sizes and small POD structs only.
 * Three layers, bottom-up:
 *
 *   1. BATCHED DEVICE API  (kvz_cuda_*_batch / *_frame, device pointers + cudaStream_t as void*)
 *      -- the throughput path: one launch evaluates many blocks / a whole frame of CTUs.
 *   2. PER-CALL STRATEGY FUNCTIONS (kvz_cuda_strat_* with the reference's exact typedefs,
 *      host pointers, synchronous) -- what the dispatch table binds; each stages its operands
 *      through a per-thread pinned buffer and runs layer 1 with count == 1.
 *   3. REGISTRARS  int kvz_strategy_register_<group>_cuda(void *opaque, uint8_t bitdepth)
 *      -- same shape as kvz_strategy_register_picture_avx2 (ref: avx2/picture-avx2.c:1718),
 *      called from kvz_strategy_register_<group>() (ref: strategies-picture.c:84-103).
 *      They call back into the host's kvz_strategyselector_register
 *      (ref: strategyselector.h:99) -- resolved at run time, see kvz_cuda_set_register_fn.
 *      Registrars for the groups whose typedefs take encoder structs (quant, sao, ipol,
 *      bipred_average) live in integration/strategies-cuda-glue.c, which is compiled
 *      against the host's headers and forwards plain parameters to this ABI.
 *
 * All functions return 0 on success and a negative KVZ_CUDA_E_* code on failure unless noted;
 * kvz_cuda_last_error() gives the message.  Every pixel argument is `const void *`:
 * uint8_t when bitdepth == 8, uint16_t when bitdepth > 8 (the reference's compile-time
 * kvz_pixel, ref: kvazaar.h:90-98).  coeff_t == int16_t (ref: global.h:115).
 */
#ifndef KVZ_CUDA_H_
#define KVZ_CUDA_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define KVZ_CUDA_PRIORITY 50           /* > avx2's 40 (ref: picture-avx2.c:1722) */
#define KVZ_CUDA_E_NODEVICE  (-1)
#define KVZ_CUDA_E_ARG       (-2)
#define KVZ_CUDA_E_RUNTIME   (-3)

/* ------------------------------------------------------------------ lifecycle */
int  kvz_cuda_init(int device);              /* idempotent; picks the device for this process */
void kvz_cuda_shutdown(void);
int  kvz_cuda_available(void);               /* 1 if a device was initialised */
const char *kvz_cuda_last_error(void);
int  kvz_cuda_sm_count(void);
/* number of kernels launched by this library since load (bench.py's gpu_launches) */
uint64_t kvz_cuda_launch_count(void);
/* event timing of the library's own launches on a stream: bracket a region */
int  kvz_cuda_sync(void *stream);

/* ------------------------------------------------------------------ 3. registrars */
typedef int (*kvz_cuda_register_fn)(void *opaque, const char *type, const char *strategy_name,
                                    int priority, void *fptr);   /* ref: strategyselector.h:99 */
/* Optional: give the callback explicitly; otherwise dlsym(RTLD_DEFAULT, "kvz_strategyselector_register"). */
void kvz_cuda_set_register_fn(kvz_cuda_register_fn fn);
int kvz_strategy_register_picture_cuda(void *opaque, uint8_t bitdepth);   /* ref: strategies-picture.h:115-227 */
int kvz_strategy_register_dct_cuda(void *opaque, uint8_t bitdepth);       /* ref: strategies-dct.h:44-82 */
int kvz_strategy_register_intra_cuda(void *opaque, uint8_t bitdepth);     /* ref: strategies-intra.h:45-75 */
int kvz_strategy_register_nal_cuda(void *opaque, uint8_t bitdepth);       /* ref: strategies-nal.h:54-68 */
int kvz_strategy_register_quant_plain_cuda(void *opaque, uint8_t bitdepth); /* coeff_abs_sum, fast_coeff_cost */
/* lookup of a per-call function by its strategy type string (what the registrars register) */
void *kvz_cuda_strategy_fptr(const char *type, uint8_t bitdepth);

/* ------------------------------------------------------------------ 2b. plain-parameter per-call entries */
/* Host pointers, synchronous; what integration/strategies-cuda-glue.c calls after unpacking encoder_state_t /
 * encoder_control_t / sao_info_t / kvz_epol_args / lcu_t (ref: strategies-quant.h:49-65, strategies-sao.h:49-68,
 * strategies-ipol.h:64-102, strategies-picture.h:136-148). */
struct kvz_cuda_quant_params_s;
void kvz_cuda_call_quant(const struct kvz_cuda_quant_params_s *p, const int16_t *coef, int16_t *q_coef, int n, int type, int scan_idx);
void kvz_cuda_call_dequant(const struct kvz_cuda_quant_params_s *p, const int16_t *q_coef, int16_t *coef, int n, int type);
int  kvz_cuda_call_quantize_residual(const struct kvz_cuda_quant_params_s *p, int width, int color, int scan_idx, int use_trskip,
                                     int cu_is_intra, int early_skip, int phase, int in_stride, int out_stride,
                                     const void *ref_in, const void *pred_in, void *rec_out, int16_t *coeff_out);
/* the same with cfg.rdoq_enable: kvz_rdoq runs on the device between the two halves; cabac = &state->cabac.ctx,
 * rp->lambda = state->lambda, tr_depth as in quant-generic.c:237-238 */
struct kvz_cuda_rdoq_params; struct kvz_cuda_cabac_ctx;
int  kvz_cuda_call_quantize_residual_rdoq(const struct kvz_cuda_quant_params_s *p, const struct kvz_cuda_rdoq_params *rp,
                                          const struct kvz_cuda_cabac_ctx *cabac, int width, int color, int scan_idx, int use_trskip,
                                          int cu_is_intra, int early_skip, int tr_depth, int in_stride, int out_stride,
                                          const void *ref_in, const void *pred_in, void *rec_out, int16_t *coeff_out);
void kvz_cuda_call_sao_edge_stats(int bitdepth, const void *orig, const void *rec, int eo_class, int bw, int bh, int *cat_sum_cnt);
int  kvz_cuda_call_sao_edge_ddistortion(int bitdepth, const void *orig, const void *rec, int bw, int bh, int eo_class, const int *offsets);
int  kvz_cuda_call_sao_band_ddistortion(int bitdepth, const void *orig, const void *rec, int bw, int bh, int band_pos, const int *bands);
void kvz_cuda_call_sao_reconstruct(int bitdepth, const void *rec_data, void *new_rec_data, int sao_type, int eo_class,
                                   const int *band_position, const int *offsets, int stride, int new_stride, int bw, int bh, int color);
void kvz_cuda_call_sample(int kind, int bitdepth, const void *src, int src_stride, int w, int h, void *dst, int dst_stride, int mvx, int mvy);
void kvz_cuda_call_filter_fme(int stage, int bitdepth, const void *src, int src_stride, int w, int h, void *filtered,
                              int16_t *hor_intermediate, int fme_level, int16_t *hor_first_cols, int hpel_off_x, int hpel_off_y);
void kvz_cuda_call_extend_block(int bitdepth, const void *src, int src_w, int src_h, int src_s, int blk_x, int blk_y, int blk_w,
                                int blk_h, int pad_l, int pad_r, int pad_t, int pad_b, int pad_b_simd, void *buf);
void kvz_cuda_call_bipred_plane(int bitdepth, void *dst, int dst_stride, const void *l0, const void *l1, int l0_is_im, int l1_is_im, int w, int h);

/* ------------------------------------------------------------------ 1. batched device API */

/* ---- picture group ---- */
/* count pairs of contiguous NxN blocks (N in 4,8,16,32,64): a[i*N*N ..], b[i*N*N ..]
 * out[i] = sad_NxN / satd_NxN of pair i (ref: picture-generic.c:475-501, 213-221, strategies-picture.h:53-69) */
int kvz_cuda_sad_nxn_batch(int n, int bitdepth, const void *a, const void *b, int count, uint32_t *out, void *stream);
int kvz_cuda_satd_nxn_batch(int n, int bitdepth, const void *a, const void *b, int count, uint32_t *out, void *stream);
/* num_modes predictions per block against one orig (dual = 2 modes, pitch 32*32, ref: picture-generic.c:363-402,
 * 512-534): pred k of block i at preds + (i*block_pitch + k*mode_pitch) pixels; costs[i*num_modes + k] */
int kvz_cuda_cost_nxn_multi_batch(int use_satd, int n, int bitdepth, const void *preds, int64_t block_pitch,
                                  int mode_pitch, int num_modes, const void *orig, int count, uint32_t *costs,
                                  void *stream);

typedef struct {           /* one strided block pair inside two planes */
  int32_t off_a, off_b;    /* pixel offsets of the top-left samples */
  int16_t w, h;
  int16_t left, right;     /* hor_sad only */
} kvz_cuda_blk;
#define KVZ_CUDA_OP_REG_SAD   0   /* ref: picture-generic.c:98-111  (no bit-depth shift) */
#define KVZ_CUDA_OP_SATD_ANY  1   /* ref: strategies-picture.h:75-113 */
#define KVZ_CUDA_OP_SSD       2   /* ref: picture-generic.c:536-551 (w x w) */
#define KVZ_CUDA_OP_VER_SAD   3   /* ref: picture-generic.c:687-701 (b = one row) */
#define KVZ_CUDA_OP_HOR_SAD   4   /* ref: picture-generic.c:714-752 */
int kvz_cuda_block_cost_batch(int op, int bitdepth, const void *plane_a, int stride_a, const void *plane_b,
                              int stride_b, const kvz_cuda_blk *descs, int count, uint32_t *out, void *stream);

typedef struct { int32_t off_pred[4]; int32_t off_orig; int16_t w, h; } kvz_cuda_quad;
/* ref: picture-generic.c:404-471, quirk for height % 8 == 4 reproduced; costs[i*4 + k] */
int kvz_cuda_satd_any_size_quad_batch(int bitdepth, const void *pred_base, int pred_stride, const void *orig_base,
                                      int orig_stride, const kvz_cuda_quad *descs, int count, uint32_t *costs,
                                      void *stream);
/* one plane of bipred_average (ref: picture-generic.c:553-668): l0/l1 contiguous w*h, pixel or int16 intermediate */
int kvz_cuda_bipred_average_plane(int bitdepth, void *dst, int dst_stride, const void *l0, const void *l1,
                                  int l0_is_im, int l1_is_im, int w, int h, void *stream);
/* pixel_var (ref: picture-generic.c:755-778) of `count` contiguous arrays of `len` pixels; sequential double sums */
int kvz_cuda_pixel_var_batch(int bitdepth, const void *buf, uint32_t len, int count, double *out, void *stream);

/* ---- dct group (ref: dct-generic.c:579-629) ---- */
#define KVZ_CUDA_TR_DCT  0
#define KVZ_CUDA_TR_IDCT 1
#define KVZ_CUDA_TR_DST  2   /* 4x4 only */
#define KVZ_CUDA_TR_IDST 3
int kvz_cuda_transform_batch(int kind, int n, int bitdepth, const int16_t *in, int16_t *out, int count, void *stream);

/* ---- quant group (ref: quant-generic.c) ---- */
typedef struct kvz_cuda_quant_params_s {
  int32_t qp;               /* state->qp */
  int32_t bitdepth;         /* encoder->bitdepth */
  int32_t slice_is_intra;   /* state->frame->slicetype == KVZ_SLICE_I */
  int32_t signhide_enable;  /* encoder->cfg.signhide_enable */
  int32_t scaling_list_enable; /* must be 0: flat lists only (all BASELINE configs) */
} kvz_cuda_quant_params;
/* count blocks of n x n coefficients; type 0 luma / 2 chroma(quant) / 2,3 chroma(dequant); scan_idx per block or NULL=0 */
int kvz_cuda_quant_batch(const kvz_cuda_quant_params *p, const int16_t *coef, int16_t *q_coef, int n, int type,
                         const int8_t *scan_idx, int count, void *stream);
int kvz_cuda_dequant_batch(const kvz_cuda_quant_params *p, const int16_t *q_coef, int16_t *coef, int n, int type,
                           int count, void *stream);
typedef struct {
  int32_t off_ref, off_pred, off_rec;  /* pixel offsets into the three planes */
  int32_t off_coeff;                   /* coeff_t offset into coeff_out */
  uint8_t width;                       /* 4,8,16,32 */
  uint8_t color;                       /* 0 Y, 1 U, 2 V */
  uint8_t scan_idx, use_trskip, cu_is_intra, early_skip;
  uint8_t phase;                       /* 0 whole function; 1 residual+forward transform only (coefficients to
                                          coeff_out, no quantisation); 2 dequant+inverse+reconstruct only (coeff_out
                                          holds the quantised levels).  Phases 1/2 bracket the host's kvz_rdoq. */
  uint8_t tr_depth;                    /* RDOQ only: cur_cu->tr_depth - cur_cu->depth (+1 for NxN), quant-generic.c:237 */
} kvz_cuda_tu;
/* kvz_quantize_residual, RDOQ-off branch (ref: quant-generic.c:198-292): residual -> DCT/DST/trskip -> quant ->
 * has_coeffs -> dequant -> inverse -> rec = clip(pred + res).  has_coeffs[i] in {0,1}. */
int kvz_cuda_quantize_residual_batch(const kvz_cuda_quant_params *p, const void *ref_plane, const void *pred_plane,
                                     int in_stride, void *rec_plane, int out_stride, int16_t *coeff_out,
                                     const kvz_cuda_tu *tus, int count, int32_t *has_coeffs, void *stream);
int kvz_cuda_coeff_abs_sum_batch(const int16_t *coeffs, size_t length, int count, uint32_t *out, void *stream);
/* returns the integer sum (the reference returns sum / 256.0) */
int kvz_cuda_fast_coeff_cost_batch(const int16_t *coeffs, int width, uint64_t weights, int count, uint32_t *out,
                                   void *stream);

/* ---- intra group (ref: intra-generic.c, intra.c:176-302) ---- */
/* level 0: the three dispatched kernels (mode 0 planar, 1 filtered DC, 2..34 angular) on the refs as given.
 * level 1: kvz_intra_predict semantics (reference smoothing, DC/edge post filters, color). */
int kvz_cuda_intra_predict_batch(int level, int log2_width, int color, int filter_boundary, int bitdepth,
                                 const void *ref_top, const void *ref_left /* [count][2w+1] */,
                                 const int8_t *modes, int count, void *dst /* [count][w*w] */, void *stream);
/* kvz_intra_build_reference over a frame-level reconstruction plane (ref: intra.c:305-559) */
int kvz_cuda_intra_build_reference_batch(int log2_width, int color, int bitdepth, const void *rec_plane, int stride,
                                         int pic_w, int pic_h, const int32_t *luma_xy /* [count][2] */, int count,
                                         void *out_top, void *out_left, void *stream);
/* Fused frame-level rough intra search (the search_intra_rough inner loop, ref: search_intra.c:391-530, batched
 * for every block of the frame): for each width-w block of the luma plane, build refs from rec_plane, predict
 * all 35 modes (kvz_intra_predict semantics, filter_boundary=1) and cost them with satd_NxN against src_plane.
 * costs: [num_blocks][35] in raster order of blocks. */
int kvz_cuda_intra_rough_search_frame(int log2_width, int bitdepth, const void *src_plane, const void *rec_plane,
                                      int stride, int pic_w, int pic_h, uint32_t *costs, void *stream);

/* ---- ipol group (ref: ipol-generic.c) ---- */
typedef struct { int32_t off_src, off_dst; int16_t w, h; int16_t mvx, mvy; } kvz_cuda_ipol;
#define KVZ_CUDA_IPOL_LUMA 0
#define KVZ_CUDA_IPOL_LUMA_HI 1
#define KVZ_CUDA_IPOL_CHROMA 2
#define KVZ_CUDA_IPOL_CHROMA_HI 3
int kvz_cuda_sample_batch(int kind, int bitdepth, const void *src_plane, int src_stride, void *dst_base,
                          int dst_stride, const kvz_cuda_ipol *descs, int count, void *stream);
#define KVZ_CUDA_IPOL_IM_SIZE ((71 + 1) * 64 + 1)  /* KVZ_IPOL_MAX_IM_SIZE_LUMA_SIMD, ref: strategies-ipol.h:53 */
#define KVZ_CUDA_IPOL_FIRST_COLS (71 + 1)
/* FME stage 0..3 = hpel hor/ver, hpel diag, qpel hor/ver, qpel diag (ref: ipol-generic.c:213-679) for `count`
 * blocks; per-block state arrays filtered[4][64*64], hor_intermediate[5][IM_SIZE], hor_first_cols[5][FIRST_COLS] */
int kvz_cuda_filter_fme_batch(int stage, int bitdepth, const void *src_plane, int src_stride, const int32_t *src_off,
                              int w, int h, void *filtered, int16_t *hor_intermediate, int fme_level,
                              int16_t *hor_first_cols, const int8_t *hpel_off /* [count][2] */, int count,
                              void *stream);
/* border-replicated copy of (blk + padding) into buf (ref: ipol-generic.c:761-814), always built */
int kvz_cuda_extend_block(int bitdepth, const void *src, int src_w, int src_h, int src_s, int blk_x, int blk_y,
                          int blk_w, int blk_h, int pad_l, int pad_r, int pad_t, int pad_b, int pad_b_simd, void *buf,
                          void *stream);

/* ---- sao group (ref: sao-generic.c, sao_shared_generics.h) ---- */
typedef struct {
  int32_t off_orig, off_rec;
  int16_t bw, bh;
  int32_t stride_orig, stride_rec;   /* 0 = contiguous copy (stride == bw), what sao.c:605-669 hands to the strategies */
} kvz_cuda_sao_blk;
/* all four EO classes at once: out[i][eo][2][5] */
int kvz_cuda_sao_edge_stats_batch(int bitdepth, const void *orig, const void *rec, const kvz_cuda_sao_blk *blks,
                                  int count, int32_t *cat_sum_cnt, void *stream);
/* offsets[i][5]; eo_class[i] */
int kvz_cuda_sao_edge_ddistortion_batch(int bitdepth, const void *orig, const void *rec, const kvz_cuda_sao_blk *blks,
                                        const int8_t *eo_class, const int32_t *offsets, int count, int32_t *out,
                                        void *stream);
int kvz_cuda_sao_band_ddistortion_batch(int bitdepth, const void *orig, const void *rec, const kvz_cuda_sao_blk *blks,
                                        const int32_t *band_pos, const int32_t *bands /* [i][4] */, int count,
                                        int32_t *out, void *stream);
typedef struct {
  int32_t off_rec, off_new;       /* pixel offsets (rec may be read 1 px around the block for edge types) */
  int16_t bw, bh;
  int8_t  type;                   /* 0 none(copy), 1 band, 2 edge  (ref: sao.h sao_type) */
  int8_t  eo_class, color, pad;
  int32_t band_position[2];
  int32_t offsets[10];
} kvz_cuda_sao_rec;
int kvz_cuda_sao_reconstruct_batch(int bitdepth, const void *rec, int stride, void *new_rec, int new_stride,
                                   const kvz_cuda_sao_rec *descs, int count, void *stream);

/* ---- nal group (ref: nal-generic.c:57-82) ---- */
/* out4: 4 bytes, big-endian checksum, device memory */
int kvz_cuda_array_checksum(int bitdepth, const void *data, int height, int width, int stride, uint8_t *out4,
                            void *stream);

/* ------------------------------------------------------------------ frame-level pass (framepass.cu) */
/* Every strategy kernel of an all-intra frame, batched over all CTUs and all four quadtree depths
 * (luma block width 32,16,8,4 = depth index 0..3; chroma width/2 for depth 0..2): rough search of 35 modes ->
 * best mode -> prediction + quantize_residual reconstruction (kvz_quant or kvz_rdoq; optional transform-skip choice
 * for 4x4 luma) + SSD + CABAC bit cost of the levels, then deblocking, SAO statistics/decision/reconstruction on the
 * 8x8-level reconstruction and the picture checksum.  Planar I420 frames, bitdepth 8 (uint8 samples) or 10 (uint16). */
typedef struct {
  int32_t width, height, bitdepth, qp, signhide;
  int32_t rdoq;      /* cfg.rdoq_enable: quantise with kvz_rdoq (slice-initial context models) instead of kvz_quant */
  int32_t trskip;    /* cfg.trskip_enable: 4x4 luma TUs also try transform skip (kvz_quantize_residual_trskip, transform.c:241-288) */
  int32_t pad;
  double  lambda;    /* state->lambda for RDOQ; 0 = the reference's constant-QP value 0.57 * 2^((qp - 12) / 3) (rate_control.c:678-691) */
} kvz_cuda_fp_params;
typedef struct {
  int32_t nblk[4];                 /* blocks per depth: (W / w) * (H / w) */
  int32_t nctu;                    /* 64x64 CTUs (partial ones included) */
  uint64_t host_bytes;             /* size of the result blob the host receives */
  /* byte offsets inside the result blob */
  uint64_t mode_y[4];              /* int8   [nblk]  best intra mode */
  uint64_t cost_y[4];              /* uint32 [nblk]  its SATD cost */
  uint64_t has_y[4];               /* uint8  [nblk]  has_coeffs */
  uint64_t ssd_y[4];               /* uint32 [nblk]  SSD(src, rec) */
  uint64_t coeff_y[4];             /* int16  [nblk][w*w] quantised coefficients, block-contiguous */
  uint64_t has_u[3], has_v[3], ssd_u[3], ssd_v[3], coeff_u[3], coeff_v[3];
  uint64_t sao_stats;              /* int32 [3*nctu][4][2][5]  (plane-major: Y CTUs, U CTUs, V CTUs) */
  uint64_t sao_dd;                 /* int32 [4][3*nctu] edge delta-distortion per class */
  uint64_t sao_band_dd;            /* int32 [3*nctu] */
  uint64_t sao_best;               /* int8  [3*nctu] chosen class or -1 */
  uint64_t sao_rec;                /* pixels: SAO-filtered I420 frame */
  uint64_t checksum;               /* 3 x 4 bytes, big-endian, Y U V */
  uint64_t bits_y[4];              /* double [nblk]  CABAC bit cost of the block's quantised coefficients (kvz_get_coeff_cost) */
  uint64_t bits_u[3], bits_v[3];
  uint64_t trskip_y;               /* uint8 [nblk[3]]  1 = the 4x4 luma TU uses transform skip (0 everywhere without params.trskip) */
  /* the coefficient sections sit together at the end of the blob: [coeff_begin, host_bytes) */
  uint64_t coeff_begin;
  /* compact form of that region (kvz_cuda_fp_run_host_compact): 32-byte chunks, one bitmap bit per chunk */
  uint64_t n_chunks;               /* (host_bytes - coeff_begin) / 32 */
  uint64_t compact_header_bytes;   /* 256 + bitmap, = offset of the packed chunks inside the compact buffer */
} kvz_cuda_fp_layout;
typedef struct kvz_cuda_frame_pass kvz_cuda_frame_pass;
kvz_cuda_frame_pass *kvz_cuda_fp_create(const kvz_cuda_fp_params *p);   /* NULL on failure */
void   kvz_cuda_fp_destroy(kvz_cuda_frame_pass *fp);
int    kvz_cuda_fp_layout_get(const kvz_cuda_frame_pass *fp, kvz_cuda_fp_layout *out);
int    kvz_cuda_fp_layout_for(const kvz_cuda_fp_params *p, kvz_cuda_fp_layout *out);   /* no device needed */
void  *kvz_cuda_fp_result_dev(kvz_cuda_frame_pass *fp);                 /* device address of the result blob */
size_t kvz_cuda_fp_frame_bytes(const kvz_cuda_frame_pass *fp);          /* W*H*3/2 */
/* frames already in HBM; rec_in_dev = reconstruction the references are taken from (NULL = the source) */
int    kvz_cuda_fp_run_dev(kvz_cuda_frame_pass *fp, const void *src_dev, const void *rec_in_dev, void *stream);
/* Per-stage device timing with CUDA events on the launching stream.  Stage index: depth d = 0..3 -> 9*d + {0 rough
 * search (+ mode selection), 1 luma recon (fused, or its forward half with RDOQ), 2 luma RDOQ, 3 luma inverse half,
 * 4 luma coefficient bit cost, 5 chroma forward (U+V), 6 chroma RDOQ (U+V), 7 chroma inverse (U+V), 8 chroma bit cost
 * (U+V)}; 36 deblocking (2 passes), 37 SAO statistics + decisions, 38 SAO reconstruction, 39 checksums.  get_timing
 * returns accumulated ms per stage over `runs` runs. */
#define KVZ_CUDA_FP_STAGES 40
int    kvz_cuda_fp_set_timing(kvz_cuda_frame_pass *fp, int enable);
int    kvz_cuda_fp_get_timing(kvz_cuda_frame_pass *fp, double *ms_total /* [KVZ_CUDA_FP_STAGES] */, int *runs);
/* Compact result: quantised coefficients are ~99 % zeros, so the coefficient region travels as a bitmap (bit c set =
 * 32-byte chunk c of [coeff_begin, host_bytes) holds a non-zero value) plus the non-zero chunks back to back, in chunk
 * order.  small_host receives blob[0, coeff_begin); compact_host receives
 *   uint32 nonzero_chunks, uint32 n_chunks, uint32 chunks_copied, pad to 256 | bitmap (n_chunks / 8, padded) | chunks
 * and must hold compact_header_bytes + budget_chunks * 32 bytes.  If nonzero_chunks > budget_chunks the tail stays on
 * the device (kvz_cuda_fp_result_dev() + host_bytes' compact region; fetch with kvz_cuda_fp_compact_fetch).  Lossless:
 * tests/test_framepass.py rebuilds the full region from it. */
int    kvz_cuda_fp_run_host_compact(kvz_cuda_frame_pass *fp, const void *src_host, void *small_host, void *compact_host,
                                    uint32_t budget_chunks, void *stream);
/* Host-side inverse (plain CPU code, no device needed): rebuild blob[coeff_begin, host_bytes) -- n_chunks * 32 bytes --
 * from a compact buffer.  Returns 0, or KVZ_CUDA_E_ARG when the buffer holds fewer chunks than the bitmap names
 * (fetch the tail first). */
int    kvz_cuda_fp_expand_compact(const kvz_cuda_fp_layout *layout, const void *compact_host, size_t compact_bytes, void *coeff_region_out);
int    kvz_cuda_fp_compact_fetch(kvz_cuda_frame_pass *fp, uint32_t first_chunk, uint32_t count, void *dst_host, void *stream);
/* host frame in (pinned for async), result blob out (host_bytes): H2D + pass + D2H enqueued on `stream` */
int    kvz_cuda_fp_run_host(kvz_cuda_frame_pass *fp, const void *src_host, void *result_host, void *stream);

/* ------------------------------------------------------------------ frame-level INTER pass (interpass.cu) */
/* Every 16x16 luma PU at least one PU away from the picture border: integer full search (+-search_range, SAD),
 * search_frac-style fractional search (hpel/qpel filter stages + SATD), motion compensation (luma 1/4, chroma 1/8
 * pel) and inter residual coding + SSD, against one reference frame.  I420, 8-bit. */
typedef struct { int32_t width, height, bitdepth, qp, search_range; } kvz_cuda_ip_params;
typedef struct {
  int32_t npu, pus_x, pus_y;        /* active PUs: pus_x * pus_y, PU (i % pus_x + 1, i / pus_x + 1) of the 16x16 grid */
  uint64_t host_bytes;
  uint64_t mv_int;                  /* int16 [npu][2]  integer MV (x, y), full-pel */
  uint64_t sad_int;                 /* uint32[npu]     its SAD */
  uint64_t mv_final;                /* int16 [npu][2]  final MV, quarter-pel */
  uint64_t satd_best;               /* uint32[npu]     its SATD */
  uint64_t has_y, ssd_y, coeff_y;   /* int32[npu], uint32[npu], int16[npu][256] */
  uint64_t has_u, has_v, ssd_u, ssd_v, coeff_u, coeff_v;   /* chroma: int16[npu][64] */
  uint64_t rec;                     /* reconstructed I420 frame (PUs outside the active area stay 0) */
} kvz_cuda_ip_layout;
typedef struct kvz_cuda_inter_pass kvz_cuda_inter_pass;
kvz_cuda_inter_pass *kvz_cuda_ip_create(const kvz_cuda_ip_params *p);
void  kvz_cuda_ip_destroy(kvz_cuda_inter_pass *ip);
int   kvz_cuda_ip_layout_for(const kvz_cuda_ip_params *p, kvz_cuda_ip_layout *out);   /* no device needed */
void *kvz_cuda_ip_result_dev(kvz_cuda_inter_pass *ip);
int   kvz_cuda_ip_run_dev(kvz_cuda_inter_pass *ip, const void *cur_dev, const void *ref_dev, void *stream);
int   kvz_cuda_ip_run_host(kvz_cuda_inter_pass *ip, const void *cur_host, const void *ref_host, void *result_host, void *stream);

/* ------------------------------------------------------------------ integer motion estimation (me_search.cu) */
/* SURVEY §8f rank 4.  The integer stage of search_pu_inter_ref (src/search_inter.c:1349-1383) for a batch of PUs
 * against one reference picture, decision for decision as the reference takes them:
 *     select_starting_point   search_inter.c:297-330   (0-vector, the predicted start MV, the merge candidates)
 *     early_terminate         search_inter.c:436-485
 *     hexagon_search          search_inter.c:712-792   (ime_algorithm = KVZ_IME_HEXBS)
 *     diamond_search          search_inter.c:812-888   (KVZ_IME_DIA)
 *     tz_search               search_inter.c:623-697   (KVZ_IME_TZ; kvz_tz_pattern_search :486-604)
 *     search_mv_full          search_inter.c:891-964   (KVZ_IME_FULL, FULL8 .. FULL64)
 * every point through check_mv_cost (search_inter.c:202-247): the tile / WPP MV constraints of
 * fracmv_within_tile (:94-181), kvz_image_calc_sad (src/image.c:407-447; references outside the picture read the
 * edge pixels, image.c:279-398), and calc_mvd_cost (:394-433) with get_mvd_coding_cost (:333-348, cfg.mv_rdo = 0)
 * over the two AMVP candidates (select_mv_cand :351-391).  The AMVP / merge candidates of a PU depend on the CUs
 * coded before it; the caller passes them in (kvz_inter_get_mv_cand / kvz_inter_get_merge_cand, src/inter.c). */
typedef struct kvz_cuda_me_params {
  int32_t width, height;            /* luma size of the (tile's) frame: state->tile->frame->width / height */
  int32_t bitdepth;                 /* 8 or 10 (pixels are uint8_t / uint16_t) */
  int32_t ime_algorithm;            /* enum kvz_ime_algorithm (kvazaar.h:110-119): hexbs, tz, full, full8..64, dia */
  int32_t me_max_steps;             /* cfg.me_max_steps (uint32; -1 = unlimited) */
  int32_t me_early_termination;     /* enum kvz_me_early_termination: 0 off, 1 on, 2 sensitive */
  int32_t mv_constraint;            /* enum kvz_mv_constraint (0 none ... 4 frame and tile with margin) */
  int32_t wpp_owf;                  /* cfg.owf && cfg.wpp: MVs may only reach LCUs that are final in the reference */
  int32_t delay_px;                 /* SAO_DELAY_PX (10) with SAO, else DEBLOCK_DELAY_PX (8) with deblocking, else 0 */
  int32_t max_ref_lcu_right, max_ref_lcu_down;   /* encoder_control_t.max_inter_ref_lcu */
  int32_t satd_final;               /* cfg.fme_level == 0: the winner's cost is recomputed with kvz_image_calc_satd (search_inter.c:1385-1397) */
  double  lambda_sqrt;              /* state->lambda_sqrt */
} kvz_cuda_me_params;
typedef struct kvz_cuda_me_merge { int16_t mv[2][2]; uint8_t dir; uint8_t ref[2]; uint8_t pad; } kvz_cuda_me_merge;   /* inter_merge_cand_t (src/inter.h:47-52): mv[list][x/y] (1/4 pel), dir, ref[list] */
typedef struct kvz_cuda_me_pu {
  int16_t x, y;                     /* info->origin (luma, tile-relative = frame-relative here) */
  int16_t w, h;                     /* info->width / height */
  int16_t mv_cand[2][2];            /* info->mv_cand (1/4 pel) */
  int16_t start_mv[2];              /* the MV the search starts from (1/4 pel): mv_previous of search_inter.c:1284-1338, or 0 */
  int16_t num_merge;                /* info->num_merge_cand, <= 5 */
  int16_t pad;
  kvz_cuda_me_merge merge[5];       /* info->merge_cand */
} kvz_cuda_me_pu;
typedef struct kvz_cuda_me_result {
  double  cost;                     /* best_cost (SAD + bits * lambda_sqrt); 1.7e308 (MAX_DOUBLE) if no point was allowed */
  int32_t bits;                     /* best_bits; INT32_MAX if no point was allowed */
  int16_t mv[2];                    /* best_mv, 1/4 pel */
  int32_t points;                   /* points whose SAD was computed (diagnostic) */
  int32_t pad;
} kvz_cuda_me_result;
/* 0 if the parameters are inside what the device search covers */
int kvz_cuda_me_params_supported(const kvz_cuda_me_params *p);
/* cur / ref: luma planes in device memory (stride in pixels); pus / out: device memory, `count` records. */
int kvz_cuda_me_search_batch(const kvz_cuda_me_params *p, const void *cur_dev, int cur_stride, const void *ref_dev, int ref_stride,
                             const kvz_cuda_me_pu *pus_dev, int count, kvz_cuda_me_result *out_dev, void *stream);
/* host buffers; synchronous */
int kvz_cuda_call_me_search(const kvz_cuda_me_params *p, const void *cur, int cur_stride, const void *ref, int ref_stride,
                            const kvz_cuda_me_pu *pus, int count, kvz_cuda_me_result *out);

/* Fractional search (search_frac, src/search_inter.c:974-1168) of a batch of PUs: half-pel, then quarter-pel positions
 * around pus[i].start_mv (= the integer search's best MV), `fme_level` (cfg.fme_level, 1..4) of the reference's four
 * steps; Hadamard costs as kvz_satd_any_size / kvz_satd_any_size_quad give them, MV cost and MV limits as above.
 * Result: best_mv (1/4 pel), best_cost, best_bits as search_frac returns them. */
int kvz_cuda_me_frac_search_batch(const kvz_cuda_me_params *p, int fme_level, const void *cur_dev, int cur_stride, const void *ref_dev, int ref_stride,
                                  const kvz_cuda_me_pu *pus_dev, int count, kvz_cuda_me_result *out_dev, void *stream);
int kvz_cuda_call_me_frac_search(const kvz_cuda_me_params *p, int fme_level, const void *cur, int cur_stride, const void *ref, int ref_stride,
                                 const kvz_cuda_me_pu *pus, int count, kvz_cuda_me_result *out);

/* Merge analysis of search_pu_inter (src/search_inter.c:1667-1730, the rdo < 3 form): every merge candidate of a PU that
 * passes the checks (bi-prediction allowed and PU larger than 8x4 / 4x8, MVs inside the limits, not a duplicate of an
 * accepted one: merge_candidate_in_list :1575-1594) is predicted -- kvz_inter_pred_pu luma, src/inter.c:604-668: one
 * list through kvz_sample_quarterpel_luma or a copy, two lists through the 14-bit samples and kvz_bipred_average --
 * and costed: kvz_satd_any_size + (merge flag bits + merge_idx + merge index bin bits) * lambda_sqrt; the accepted
 * candidates come back sorted by cost (kvz_sort_keys_by_cost, src/search.c:612-626).  The early-skip reconstruction
 * that follows in the reference (:1735-1790) is not part of this entry. */
typedef struct kvz_cuda_me_refs {
  const void *plane[16];            /* luma planes of state->frame->ref->images[i] in device memory (stride = their width) */
  int32_t stride[16];
  uint8_t ref_LX[2][16];            /* state->frame->ref_LX: list index -> picture index */
  int32_t bipred;                   /* cfg.bipred */
  int32_t pad;
  double merge_flag_bits;           /* CTX_ENTROPY_FBITS(search_cabac.ctx.cu_merge_flag_ext_model, 1) */
  double merge_idx_bits[2];         /* CTX_ENTROPY_FBITS(search_cabac.ctx.cu_merge_idx_ext_model, 0 / 1) */
} kvz_cuda_me_refs;
typedef struct kvz_cuda_me_merge_cost {
  double cost[5], bits[5];          /* per accepted candidate, in acceptance order; unused entries 1.7e308 / 0 */
  int32_t size;                     /* accepted candidates */
  int8_t keys[5];                   /* acceptance-order indices sorted by ascending cost; unused -1 */
  int8_t merge_idx[5];              /* merge index of each accepted candidate */
  int8_t pad[2];
} kvz_cuda_me_merge_cost;
int kvz_cuda_me_merge_cost_batch(const kvz_cuda_me_params *p, const kvz_cuda_me_refs *refs, const void *cur_dev, int cur_stride,
                                 const kvz_cuda_me_pu *pus_dev, int count, kvz_cuda_me_merge_cost *out_dev, void *stream);

/* Bi-prediction from the best uni-predictions of the two lists (search_pu_inter, src/search_inter.c:1937-2031, the
 * cfg.fast_bipred path every preset uses): kvz_inter_recon_bipred luma + kvz_satd_any_size, the MV costs of both MVs
 * against info->mv_cand (calc_mvd_cost, mv_shift 0), reference-index and direction bits, and select_mv_cand for each
 * list.  The caller passes the MVs / reference indices of the two uni-predictions and the AMVP candidates info->mv_cand
 * holds at that point (those of list 1: kvz_cuda_me_candidates_batch with the PU's mv_ref). */
typedef struct kvz_cuda_me_bipred_pu {
  int16_t x, y, w, h;
  int16_t mv[2][2];                 /* best_unipred[0]->inter.mv[0], best_unipred[1]->inter.mv[1] (1/4 pel) */
  uint8_t mv_ref[2];                /* their reference indices in L0 / L1 */
  uint8_t pad[2];
  int16_t mv_cand[2][2];            /* info->mv_cand */
} kvz_cuda_me_bipred_pu;
typedef struct kvz_cuda_me_bipred_result {
  double  cost;                     /* best_bipred_cost; 1.7e308 when bi-prediction may not be used (cfg.bipred off, w + h < 16) */
  int32_t bits;                     /* bitcost[0] + bitcost[1] + extra_bits */
  uint8_t mv_cand_idx[2];           /* CU_SET_MV_CAND of each list */
  uint8_t valid, pad;
} kvz_cuda_me_bipred_result;
int kvz_cuda_me_bipred_batch(const kvz_cuda_me_params *p, const kvz_cuda_me_refs *refs, const void *cur_dev, int cur_stride,
                             const kvz_cuda_me_bipred_pu *pus_dev, int count, kvz_cuda_me_bipred_result *out_dev, void *stream);

/* Motion compensation of a batch of decided PUs (kvz_inter_pred_pu, src/inter.c:604-668, luma and chroma): one list through
 * kvz_sample_quarterpel_luma / kvz_sample_octpel_chroma (or the plain copy for integer MVs), two lists through the 14-bit
 * samples and kvz_bipred_average; reference samples outside the picture are the edge samples.  The prediction is written
 * into an I420 picture (the PUs of a batch must not overlap). */
typedef struct kvz_cuda_me_mc_refs {
  const void *y[16], *u[16], *v[16];   /* planes of state->frame->ref->images[i] in device memory; luma stride = width, chroma width / 2 */
  uint8_t ref_LX[2][16];
} kvz_cuda_me_mc_refs;
typedef struct kvz_cuda_me_mc_pu {
  int16_t x, y, w, h;               /* luma samples; multiples of 4 */
  int16_t mv[2][2];                 /* inter.mv[list] (1/4 pel) */
  uint8_t mv_ref[2];                /* inter.mv_ref[list] */
  uint8_t dir;                      /* inter.mv_dir: 1, 2 or 3 */
  uint8_t pad;
} kvz_cuda_me_mc_pu;
int kvz_cuda_me_predict_batch(const kvz_cuda_me_params *p, const kvz_cuda_me_mc_refs *refs, const kvz_cuda_me_mc_pu *pus_dev, int count,
                              void *pred_y_dev, void *pred_u_dev, void *pred_v_dev, void *stream);

/* AMVP and merge candidates of a batch of PUs from a snapshot of the CU records (me_search.cu), as
 *     kvz_inter_get_mv_cand_cua   src/inter.c:1365-1383 (get_spatial_merge_candidates_cua :1015-1076,
 *                                 get_temporal_merge_candidates :836-907, get_mv_cand_from_candidates :1225-1318,
 *                                 add_mvp_candidate :1186-1220, apply_mv_scaling_pocs :1084-1103, add_temporal_candidate :1134-1184)
 *     kvz_inter_get_merge_cand    src/inter.c:1440-1572 (is_a0/b0_cand_coded :689-823, add_merge_candidate :1403-1425)
 * derive them.  In the encoder the neighbours of a PU are the CUs decided before it, so a caller uses this for PUs
 * whose neighbourhood is final (the rows above, a previous pass, the colocated picture); the result feeds
 * kvz_cuda_me_search_batch. */
typedef struct kvz_cuda_me_cu {       /* the fields of cu_info_t (src/cu.h:126-165) the derivation reads; one record per 4x4 luma block */
  int16_t mv[2][2];                   /* inter.mv[list][x/y] */
  uint8_t type;                       /* cu_type_t: 0 not set, 1 intra, 2 inter */
  uint8_t mv_dir;                     /* 1 = L0, 2 = L1, 3 = both */
  uint8_t mv_ref[2];                  /* index into L0 / L1 */
} kvz_cuda_me_cu;
typedef struct kvz_cuda_me_frame {    /* state->frame / state->frame->ref as the derivation reads them */
  int32_t width, height;              /* encoder_control->in.width / height (= the tile frame here) */
  int32_t poc;                        /* state->frame->poc */
  int32_t slice_b;                    /* state->frame->slicetype == KVZ_SLICE_B */
  int32_t tmvp_enable, max_merge;     /* cfg.tmvp_enable, cfg.max_merge */
  int32_t used_size;                  /* state->frame->ref->used_size */
  int32_t ref_LX_size[2];             /* state->frame->ref_LX_size */
  int32_t pocs[16];                   /* state->frame->ref->pocs */
  int32_t col_ref_pocs[2][16];        /* for the colocated picture c = ref_LX[0][0]: images[c]->ref_pocs[ref_LXs[c][list][mv_ref]] */
  uint8_t ref_LX[2][16];              /* state->frame->ref_LX */
} kvz_cuda_me_frame;
typedef struct kvz_cuda_me_cand_pu {
  int16_t x, y, w, h;                 /* the PU, luma samples */
  uint8_t mv_ref[2];                  /* cur_cu->inter.mv_ref[list]: the reference index the AMVP of each list is derived for */
  uint8_t use_a1, use_b1;             /* merge: may A1 / B1 be used (false for the second PU of Nx2N / 2NxN, search_inter.c:1628-1633) */
} kvz_cuda_me_cand_pu;
typedef struct kvz_cuda_me_cand_out {
  int16_t mv_cand[2][2][2];           /* [list][candidate][x/y]; list 1 is zero when L1 is empty */
  int32_t num_merge;
  kvz_cuda_me_merge merge[5];         /* unused entries and fields the reference leaves unset are 0 */
} kvz_cuda_me_cand_out;
/* cus / col_cus: CU records of the current and of the colocated picture in device memory, `stride` records per row */
int kvz_cuda_me_candidates_batch(const kvz_cuda_me_frame *f, const kvz_cuda_me_cu *cus_dev, int cu_stride, const kvz_cuda_me_cu *col_cus_dev,
                                 int col_stride, const kvz_cuda_me_cand_pu *pus_dev, int count, kvz_cuda_me_cand_out *out_dev, void *stream);
/* host buffers; synchronous.  cu_rows = rows of both CU images */
int kvz_cuda_call_me_candidates(const kvz_cuda_me_frame *f, const kvz_cuda_me_cu *cus, int cu_stride, const kvz_cuda_me_cu *col_cus, int col_stride,
                                int cu_rows, const kvz_cuda_me_cand_pu *pus, int count, kvz_cuda_me_cand_out *out);

/* ------------------------------------------------------------------ host-buffer conveniences */
/* ---------------------------------------------------------------------------------------------------------
 * RDOQ (SURVEY §8f rank 1): kvz_rdoq (src/rdo.c:661-977) incl. kvz_rdoq_sign_hiding (rdo.c:518-653) and the
 * find_last_scanpos strategy (quant-generic.c:376-399), flat scaling lists.
 * The CABAC context models enter as the memory image of the reference's `cabac_data_t.ctx` member
 * (src/cabac.h:66-102: one uc_state byte per context model): a binding copies &state->cabac.ctx.
 * --------------------------------------------------------------------------------------------------------- */
typedef struct kvz_cuda_cabac_ctx {            /* field order = src/cabac.h:67-101 */
  uint8_t sao_merge_flag_model, sao_type_idx_model, split_flag_model[3], intra_mode_model, chroma_pred_model[2],
          inter_dir[5], trans_subdiv_model[3], qt_cbf_model_luma[4], qt_cbf_model_chroma[4], cu_qp_delta_abs[4],
          part_size_model[4], cu_sig_coeff_group_model[4], cu_sig_model_luma[27], cu_sig_model_chroma[15],
          cu_ctx_last_y_luma[15], cu_ctx_last_y_chroma[15], cu_ctx_last_x_luma[15], cu_ctx_last_x_chroma[15],
          cu_one_model_luma[16], cu_one_model_chroma[8], cu_abs_model_luma[4], cu_abs_model_chroma[2],
          cu_pred_mode_model, cu_skip_flag_model[3], cu_merge_idx_ext_model, cu_merge_flag_ext_model,
          cu_transquant_bypass, cu_mvd_model[2], cu_ref_pic_model[2], mvp_idx_model[2], cu_qt_root_cbf_model,
          transform_skip_model_luma, transform_skip_model_chroma;
} kvz_cuda_cabac_ctx;
/* kvz_init_contexts (src/context.c:221-304): the context models at the start of a slice.  slice_type: 0 B, 1 P, 2 I.  Host only. */
int kvz_cuda_cabac_ctx_init(int qp, int slice_type, kvz_cuda_cabac_ctx *out);
typedef struct kvz_cuda_rdoq_params {
  double  lambda;            /* state->lambda */
  int32_t qp;                /* state->qp */
  int32_t bitdepth;
  int32_t signhide_enable;   /* cfg.signhide_enable */
  int32_t pad;
} kvz_cuda_rdoq_params;
typedef struct kvz_cuda_rdoq_tu {
  int32_t off_coef;          /* coeff_t offset of the n x n transform coefficients in `coef` */
  int32_t off_dest;          /* coeff_t offset of the quantised levels in `dest` */
  uint8_t type;              /* 0 luma, 2 chroma (the reference passes 2 for U and V, quant-generic.c:239) */
  uint8_t scan_idx;          /* 0 diagonal, 1 horizontal, 2 vertical */
  uint8_t block_type;        /* cu type: 1 intra, 2 inter */
  uint8_t tr_depth;          /* cur_cu->tr_depth - cur_cu->depth (+1 for NxN), quant-generic.c:237-238 */
} kvz_cuda_rdoq_tu;
/* kvz_quantize_residual with the RDOQ branch taken (quant-generic.c:234-240) entirely on the device: residual +
 * forward transform, kvz_rdoq, dequant + inverse transform + reconstruction.  widths_mask: OR of the TU widths in
 * the batch (4 | 8 | 16 | 32).  Descriptors as for kvz_cuda_quantize_residual_batch (phase must be 0). */
int kvz_cuda_quantize_residual_rdoq_batch(const kvz_cuda_quant_params *p, const kvz_cuda_rdoq_params *rp,
                                          const kvz_cuda_cabac_ctx *ctx_dev, const void *ref_plane, const void *pred_plane,
                                          int in_stride, void *rec_plane, int out_stride, int16_t *coeff_out,
                                          const kvz_cuda_tu *tus, int count, int widths_mask, int32_t *has_coeffs, void *stream);
/* `count` TUs of width n (4, 8, 16 or 32); ctx_dev: one kvz_cuda_cabac_ctx shared by the batch */
int kvz_cuda_rdoq_batch(const kvz_cuda_rdoq_params *p, const kvz_cuda_cabac_ctx *ctx_dev, const int16_t *coef, int16_t *dest,
                        int n, const kvz_cuda_rdoq_tu *tus, int count, void *stream);

/* CABAC bit cost of quantised coefficients: the CABAC branch of kvz_get_coeff_cost (src/rdo.c:291-330), i.e.
 * kvz_encode_coeff_nxn in only_count mode (encode_coding_tree-generic.c:40-290).  Descriptors: kvz_cuda_rdoq_tu with
 * off_coef = offset of the n x n levels, type 0 luma / 2 chroma, scan_idx, and `block_type` carrying the TU's
 * transform_skip flag (only read for 4x4 with trskip_enable); off_dest / tr_depth unused.  bits_out[count] doubles.
 * update = cabac->update: the context models adapt inside each TU; ctx_out (optional, [count]) receives them. */
typedef struct kvz_cuda_coeff_cost_params {
  int32_t signhide_enable;   /* cfg.signhide_enable */
  int32_t trskip_enable;     /* cfg.trskip_enable */
  int32_t update;            /* cabac->update */
  int32_t pad;
} kvz_cuda_coeff_cost_params;
int kvz_cuda_coeff_cost_batch(const kvz_cuda_coeff_cost_params *p, const kvz_cuda_cabac_ctx *ctx_dev, const int16_t *coeff, int n,
                              const kvz_cuda_rdoq_tu *tus, int count, double *bits_out, kvz_cuda_cabac_ctx *ctx_out, void *stream);

/* ---------------------------------------------------------------------------------------------------------
 * Deblocking filter, frame level (SURVEY §8f rank 3).  Replaces the per-LCU kvz_filter_deblock_lcu
 * (src/filter.c:783-792, called from encoder_state_worker_encode_lcu_search, src/encoderstate.c:669-675) by two
 * passes over the frame (all vertical edges, then all horizontal edges) -- the same result, see csrc/deblock.cu.
 * `cus`: one 20-byte record per 4x4 SCU = the memory image of the reference's cu_info_t (src/cu.h:126-165,
 * x86-64 SysV), row stride cu_stride_scu records: a binding passes frame->cu_array->data and stride / 4.
 * Planes are filtered in place.  U/V may both be NULL (4:0:0).
 * --------------------------------------------------------------------------------------------------------- */
typedef struct kvz_cuda_dbk_params {
  int32_t width, height;           /* luma size, multiples of 8 */
  int32_t qp;                      /* state->qp, used when per_cu_qp == 0 (frame->max_qp_delta_depth < 0, filter.c:262) */
  int32_t beta_offset_div2;        /* cfg.deblock_beta */
  int32_t tc_offset_div2;          /* cfg.deblock_tc */
  int32_t slice_is_b;              /* frame->slicetype == KVZ_SLICE_B (filter.c:404) */
  int32_t per_cu_qp;               /* average the cu_info_t.qp of both sides (filter.c:268-282) */
  int32_t cu_stride_scu;           /* cu_array->stride / 4 */
  uint8_t ref_LX[2][16];           /* frame->ref_LX (src/encoderstate.h:125), B slices only */
} kvz_cuda_dbk_params;
int kvz_cuda_deblock_frame(const kvz_cuda_dbk_params *p, int bitdepth, void *y_dev, void *u_dev, void *v_dev,
                           const void *cus_dev, void *stream);
/* host buffers (kvz_picture planes with luma stride `stride`, chroma stride / 2); synchronous */
int kvz_cuda_call_deblock_frame(const kvz_cuda_dbk_params *p, int bitdepth, void *y, void *u, void *v, int stride,
                                const void *cus);

/* device memory helpers so that C hosts need no CUDA headers */
void *kvz_cuda_malloc(size_t bytes);
void  kvz_cuda_free(void *p);
void *kvz_cuda_host_alloc(size_t bytes);     /* pinned */
void  kvz_cuda_host_free(void *p);
int   kvz_cuda_memcpy_h2d(void *dst, const void *src, size_t bytes, void *stream);
int   kvz_cuda_memcpy_d2h(void *dst, const void *src, size_t bytes, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* KVZ_CUDA_H_ */
