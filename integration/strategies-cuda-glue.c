/*
 * strategies-cuda-glue.c -- the host-side ("C stays C") half of the cuda strategy.
 *
 * This file is what a Kvazaar maintainer adds under src/strategies/cuda/: it is compiled WITH the encoder's own
 * headers, so it may look inside encoder_state_t / encoder_control_t / sao_info_t / kvz_epol_args / lcu_t, and it
 * forwards plain parameters to libkvzcuda.so (include/kvz_cuda.h), which knows nothing about those structs.
 * It provides
 *   - the registrars for the struct-typed groups:  kvz_strategy_register_{quant,sao,ipol}_cuda and the
 *     bipred_average member of the picture group;
 *   - kvz_strategy_register_all_cuda(opaque, bitdepth): every group in one call;
 *   - kvz_cuda_overlay_install(): binds the cuda strategies into an ALREADY INITIALISED, unmodified libkvazaar by
 *     overwriting its exported global function pointers (SURVEY.md H7) -- used by the drop-in tests here, where the
 *     reference build may not be patched.
 * In a patched tree each kvz_strategy_register_<group>() simply calls the matching *_cuda registrar after the AVX2
 * one (ref: strategies-picture.c:84-103); see INTEGRATION.md.
 */
#include <dlfcn.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "global.h"
#include "kvazaar.h"
#include "encoder.h"
#include "encoderstate.h"
#include "strategyselector.h"
#include "cu.h"
#include "image.h"
#include "sao.h"
#include "transform.h"

#include "kvz_cuda.h"

/* ------------------------------------------------------------------------------------------------ quant group */
static void fill_qp(const encoder_state_t *state, kvz_cuda_quant_params *p)
{
  const encoder_control_t *enc = state->encoder_control;
  if (enc->scaling_list.enable) {
    fprintf(stderr, "kvz-cuda: custom scaling lists (--cqmfile) are not supported by the cuda strategy; "
                    "run with KVAZAAR_OVERRIDE_quant=avx2 KVAZAAR_OVERRIDE_dequant=avx2 KVAZAAR_OVERRIDE_quantize_residual=avx2\n");
    abort();
  }
  p->qp = state->qp;
  p->bitdepth = enc->bitdepth;
  p->slice_is_intra = state->frame->slicetype == KVZ_SLICE_I;
  p->signhide_enable = enc->cfg.signhide_enable;
  p->scaling_list_enable = 0;
}

/* ref: strategies-quant.h:49 (quant_func) */
static void quant_cuda(const encoder_state_t *const state, coeff_t *coef, coeff_t *q_coef, int32_t width, int32_t height,
                       int8_t type, int8_t scan_idx, int8_t block_type)
{
  (void)height; (void)block_type;
  kvz_cuda_quant_params p; fill_qp(state, &p);
  kvz_cuda_call_quant(&p, coef, q_coef, width, type, scan_idx);
}

/* ref: strategies-quant.h:58 (dequant_func) */
static void dequant_cuda(const encoder_state_t *const state, coeff_t *q_coef, coeff_t *coef, int32_t width, int32_t height,
                         int8_t type, int8_t block_type)
{
  (void)height; (void)block_type;
  kvz_cuda_quant_params p; fill_qp(state, &p);
  kvz_cuda_call_dequant(&p, q_coef, coef, width, type);
}

/* ref: strategies-quant.h:51-57 (quant_residual_func), quant-generic.c:198-292.  With RDOQ, kvz_rdoq (not a strategy,
 * src/rdo.c:661) runs on the device too (csrc/rdoq.cuh), between the forward and inverse halves, exactly where the
 * generic and AVX2 versions call it. */
static int quantize_residual_cuda(encoder_state_t *const state, const cu_info_t *const cur_cu, const int width,
                                  const color_t color, const coeff_scan_order_t scan_order, const int use_trskip,
                                  const int in_stride, const int out_stride, const kvz_pixel *const ref_in,
                                  const kvz_pixel *const pred_in, kvz_pixel *rec_out, coeff_t *coeff_out, bool early_skip)
{
  kvz_cuda_quant_params p; fill_qp(state, &p);
  const encoder_control_t *enc = state->encoder_control;
  const int intra = cur_cu->type == CU_INTRA;
  if (enc->cfg.rdoq_enable && (width > 4 || !enc->cfg.rdoq_skip)) {
    /* kvz_rdoq on the device: the context models and lambda it reads are state->cabac.ctx and state->lambda (rdo.c:665-884) */
    _Static_assert(sizeof(kvz_cuda_cabac_ctx) == sizeof(((cabac_data_t *)0)->ctx), "cabac ctx image");
    kvz_cuda_rdoq_params rp = { state->lambda, state->qp, enc->bitdepth, enc->cfg.signhide_enable, 0 };
    int8_t tr_depth = cur_cu->tr_depth - cur_cu->depth;
    tr_depth += (cur_cu->part_size == SIZE_NxN ? 1 : 0);
    return kvz_cuda_call_quantize_residual_rdoq(&p, &rp, (const kvz_cuda_cabac_ctx *)&state->cabac.ctx, width, color, scan_order, use_trskip,
                                                intra, early_skip, tr_depth, in_stride, out_stride, ref_in, pred_in, rec_out, coeff_out);
  }
  return kvz_cuda_call_quantize_residual(&p, width, color, scan_order, use_trskip, intra, early_skip, 0, in_stride, out_stride,
                                         ref_in, pred_in, rec_out, coeff_out);
}

/* ------------------------------------------------------------------------------------------------ sao group */
static void calc_sao_edge_dir_cuda(const encoder_control_t *const encoder, const kvz_pixel *orig_data, const kvz_pixel *rec_data,
                                   int eo_class, int block_width, int block_height, int cat_sum_cnt[2][NUM_SAO_EDGE_CATEGORIES])
{
  kvz_cuda_call_sao_edge_stats(encoder->bitdepth, orig_data, rec_data, eo_class, block_width, block_height, &cat_sum_cnt[0][0]);
}
static int sao_edge_ddistortion_cuda(const encoder_control_t *const encoder, const kvz_pixel *orig_data, const kvz_pixel *rec_data,
                                     int block_width, int block_height, int eo_class, int offsets[NUM_SAO_EDGE_CATEGORIES])
{
  return kvz_cuda_call_sao_edge_ddistortion(encoder->bitdepth, orig_data, rec_data, block_width, block_height, eo_class, offsets);
}
static int sao_band_ddistortion_cuda(const encoder_state_t *const state, const kvz_pixel *orig_data, const kvz_pixel *rec_data,
                                     int block_width, int block_height, int band_pos, const int sao_bands[4])
{
  return kvz_cuda_call_sao_band_ddistortion(state->encoder_control->bitdepth, orig_data, rec_data, block_width, block_height, band_pos, sao_bands);
}
static void sao_reconstruct_color_cuda(const encoder_control_t *const encoder, const kvz_pixel *rec_data, kvz_pixel *new_rec_data,
                                       const sao_info_t *sao, int stride, int new_stride, int block_width, int block_height, color_t color_i)
{
  kvz_cuda_call_sao_reconstruct(encoder->bitdepth, rec_data, new_rec_data, sao->type, sao->eo_class, sao->band_position, sao->offsets,
                                stride, new_stride, block_width, block_height, color_i);
}

/* ------------------------------------------------------------------------------------------------ ipol group */
#define SAMPLE_FN(name, kind, dst_t)                                                                                   \
  static void name(const encoder_control_t *const encoder, kvz_pixel *src, int16_t src_stride, int width, int height,  \
                   dst_t *dst, int16_t dst_stride, int8_t hor_flag, int8_t ver_flag, const int16_t mv[2])              \
  {                                                                                                                    \
    (void)encoder; (void)hor_flag; (void)ver_flag;                                                                     \
    kvz_cuda_call_sample(kind, KVZ_BIT_DEPTH, src, src_stride, width, height, dst, dst_stride, mv[0], mv[1]);          \
  }
SAMPLE_FN(sample_quarterpel_luma_cuda, KVZ_CUDA_IPOL_LUMA, kvz_pixel)
SAMPLE_FN(sample_quarterpel_luma_hi_cuda, KVZ_CUDA_IPOL_LUMA_HI, int16_t)
SAMPLE_FN(sample_octpel_chroma_cuda, KVZ_CUDA_IPOL_CHROMA, kvz_pixel)
SAMPLE_FN(sample_octpel_chroma_hi_cuda, KVZ_CUDA_IPOL_CHROMA_HI, int16_t)

#define FME_FN(name, stage)                                                                                            \
  static void name(const encoder_control_t *encoder, kvz_pixel *src, int16_t src_stride, int width, int height,        \
                   kvz_pixel filtered[4][LCU_LUMA_SIZE], int16_t hor_intermediate[5][KVZ_IPOL_MAX_IM_SIZE_LUMA_SIMD],  \
                   int8_t fme_level, int16_t hor_first_cols[5][KVZ_EXT_BLOCK_W_LUMA + 1], int8_t off_x, int8_t off_y)  \
  {                                                                                                                    \
    (void)encoder;                                                                                                     \
    kvz_cuda_call_filter_fme(stage, KVZ_BIT_DEPTH, src, src_stride, width, height, &filtered[0][0],                   \
                             &hor_intermediate[0][0], fme_level, &hor_first_cols[0][0], off_x, off_y);                \
  }
FME_FN(filter_hpel_blocks_hor_ver_luma_cuda, 0)
FME_FN(filter_hpel_blocks_diag_luma_cuda, 1)
FME_FN(filter_qpel_blocks_hor_ver_luma_cuda, 2)
FME_FN(filter_qpel_blocks_diag_luma_cuda, 3)

/* ref: strategies-ipol.h:68-95, ipol-generic.c:761-814.  The in-bounds case only hands out pointers. */
static void get_extended_block_cuda(kvz_epol_args *args)
{
  const int min_y = args->blk_y - args->pad_t, max_y = args->blk_y + args->blk_h + args->pad_b + args->pad_b_simd - 1;
  const int min_x = args->blk_x - args->pad_l, max_x = args->blk_x + args->blk_w + args->pad_r - 1;
  if (min_y < 0 || max_y >= args->src_h || min_x < 0 || max_x >= args->src_w) {
    *args->ext = args->buf;
    *args->ext_s = args->pad_l + args->blk_w + args->pad_r;
    *args->ext_origin = args->buf + args->pad_t * (*args->ext_s) + args->pad_l;
    kvz_cuda_call_extend_block(KVZ_BIT_DEPTH, args->src, args->src_w, args->src_h, args->src_s, args->blk_x, args->blk_y,
                               args->blk_w, args->blk_h, args->pad_l, args->pad_r, args->pad_t, args->pad_b, args->pad_b_simd, args->buf);
  } else {
    *args->ext = args->src + (args->blk_y - args->pad_t) * args->src_s + (args->blk_x - args->pad_l);
    *args->ext_origin = args->src + args->blk_y * args->src_s + args->blk_x;
    *args->ext_s = args->src_s;
  }
}

/* ------------------------------------------------------------------------------------------------ picture: bipred */
/* ref: strategies-picture.h:136-148, picture-generic.c:634-668 */
static void bipred_average_cuda(lcu_t *const lcu, const yuv_t *const px_L0, const yuv_t *const px_L1, const yuv_im_t *const im_L0,
                                const yuv_im_t *const im_L1, const unsigned pu_x, const unsigned pu_y, const unsigned pu_w,
                                const unsigned pu_h, const unsigned im_flags_L0, const unsigned im_flags_L1,
                                const bool predict_luma, const bool predict_chroma)
{
  if (predict_luma) {
    const unsigned off = SUB_SCU(pu_y) * LCU_WIDTH + SUB_SCU(pu_x);
    const int i0 = im_flags_L0 & 1, i1 = im_flags_L1 & 1;
    kvz_cuda_call_bipred_plane(KVZ_BIT_DEPTH, lcu->rec.y + off, LCU_WIDTH, i0 ? (void *)im_L0->y : (void *)px_L0->y,
                               i1 ? (void *)im_L1->y : (void *)px_L1->y, i0, i1, pu_w, pu_h);
  }
  if (predict_chroma) {
    const unsigned off = SUB_SCU(pu_y) / 2 * LCU_WIDTH_C + SUB_SCU(pu_x) / 2;
    const int i0 = (im_flags_L0 & 2) != 0, i1 = (im_flags_L1 & 2) != 0;
    kvz_cuda_call_bipred_plane(KVZ_BIT_DEPTH, lcu->rec.u + off, LCU_WIDTH_C, i0 ? (void *)im_L0->u : (void *)px_L0->u,
                               i1 ? (void *)im_L1->u : (void *)px_L1->u, i0, i1, pu_w / 2, pu_h / 2);
    kvz_cuda_call_bipred_plane(KVZ_BIT_DEPTH, lcu->rec.v + off, LCU_WIDTH_C, i0 ? (void *)im_L0->v : (void *)px_L0->v,
                               i1 ? (void *)im_L1->v : (void *)px_L1->v, i0, i1, pu_w / 2, pu_h / 2);
  }
}

/* ------------------------------------------------------------------------------------------------ registrars */
typedef struct { const char *type; void *fptr; const char *group; } glue_entry;
static const glue_entry glue_entries[] = {
  { "quant", (void *)&quant_cuda, "quant" },
  { "dequant", (void *)&dequant_cuda, "quant" },
  { "quantize_residual", (void *)&quantize_residual_cuda, "quant" },
  { "calc_sao_edge_dir", (void *)&calc_sao_edge_dir_cuda, "sao" },
  { "sao_edge_ddistortion", (void *)&sao_edge_ddistortion_cuda, "sao" },
  { "sao_band_ddistortion", (void *)&sao_band_ddistortion_cuda, "sao" },
  { "sao_reconstruct_color", (void *)&sao_reconstruct_color_cuda, "sao" },
  { "sample_quarterpel_luma", (void *)&sample_quarterpel_luma_cuda, "ipol" },
  { "sample_quarterpel_luma_hi", (void *)&sample_quarterpel_luma_hi_cuda, "ipol" },
  { "sample_octpel_chroma", (void *)&sample_octpel_chroma_cuda, "ipol" },
  { "sample_octpel_chroma_hi", (void *)&sample_octpel_chroma_hi_cuda, "ipol" },
  { "filter_hpel_blocks_hor_ver_luma", (void *)&filter_hpel_blocks_hor_ver_luma_cuda, "ipol" },
  { "filter_hpel_blocks_diag_luma", (void *)&filter_hpel_blocks_diag_luma_cuda, "ipol" },
  { "filter_qpel_blocks_hor_ver_luma", (void *)&filter_qpel_blocks_hor_ver_luma_cuda, "ipol" },
  { "filter_qpel_blocks_diag_luma", (void *)&filter_qpel_blocks_diag_luma_cuda, "ipol" },
  { "get_extended_block", (void *)&get_extended_block_cuda, "ipol" },
  { "bipred_average", (void *)&bipred_average_cuda, "picture" },
};

static int register_glue_group(void *opaque, const char *group)
{
  if (!kvz_cuda_available()) return 1;            /* no device: register nothing, keep the host's strategies */
  int ok = 1;
  for (unsigned i = 0; i < sizeof(glue_entries) / sizeof(glue_entries[0]); ++i)
    if (strcmp(glue_entries[i].group, group) == 0)
      ok &= kvz_strategyselector_register(opaque, glue_entries[i].type, "cuda", KVZ_CUDA_PRIORITY, glue_entries[i].fptr);
  return ok;
}

int kvz_strategy_register_quant_cuda(void *opaque, uint8_t bitdepth)
{
  return register_glue_group(opaque, "quant") & kvz_strategy_register_quant_plain_cuda(opaque, bitdepth);
}
int kvz_strategy_register_sao_cuda(void *opaque, uint8_t bitdepth) { (void)bitdepth; return register_glue_group(opaque, "sao"); }
int kvz_strategy_register_ipol_cuda(void *opaque, uint8_t bitdepth) { (void)bitdepth; return register_glue_group(opaque, "ipol"); }
int kvz_strategy_register_picture_all_cuda(void *opaque, uint8_t bitdepth)
{
  return kvz_strategy_register_picture_cuda(opaque, bitdepth) & register_glue_group(opaque, "picture");
}

int kvz_strategy_register_all_cuda(void *opaque, uint8_t bitdepth)
{
  int ok = 1;
  ok &= kvz_strategy_register_picture_all_cuda(opaque, bitdepth);
  ok &= kvz_strategy_register_nal_cuda(opaque, bitdepth);
  ok &= kvz_strategy_register_dct_cuda(opaque, bitdepth);
  ok &= kvz_strategy_register_ipol_cuda(opaque, bitdepth);
  ok &= kvz_strategy_register_quant_cuda(opaque, bitdepth);
  ok &= kvz_strategy_register_intra_cuda(opaque, bitdepth);
  ok &= kvz_strategy_register_sao_cuda(opaque, bitdepth);
  return ok;
}

/* ------------------------------------------------------------------------------------------------ overlay */
/* Bind into an unmodified, already initialised libkvazaar: for every registered ("type", fptr) overwrite the
 * exported global `kvz_<type>` (ref: strategyselector.h:112-122 strategies_to_select).  `only` = NULL or a
 * comma-separated list of type strings / group names to restrict the overlay (for bisecting). Returns the number
 * of pointers replaced, or -1. */
static int overlay_count;
static const char *overlay_filter;
static int overlay_cb(void *opaque, const char *type, const char *strategy_name, int priority, void *fptr)
{
  (void)opaque; (void)strategy_name; (void)priority;
  if (overlay_filter && overlay_filter[0]) {
    const size_t n = strlen(type);
    const char *p = overlay_filter;
    int hit = 0;
    while (p && *p) {
      const char *e = strchr(p, ',');
      const size_t len = e ? (size_t)(e - p) : strlen(p);
      if (len == n && strncmp(p, type, n) == 0) { hit = 1; break; }
      p = e ? e + 1 : NULL;
    }
    if (!hit) return 1;
  }
  for (const strategy_to_select_t *s = strategies_to_select; s->strategy_type; ++s) {
    if (strcmp(s->strategy_type, type) == 0) { *s->fptr = fptr; ++overlay_count; return 1; }
  }
  fprintf(stderr, "kvz-cuda overlay: the host has no strategy type '%s'\n", type);
  return 0;
}

/* kvz_strategyselector_register look-alike that the plain registrars of libkvzcuda call back into */
static int overlay_register(void *opaque, const char *type, const char *strategy_name, int priority, void *fptr)
{
  return overlay_cb(opaque, type, strategy_name, priority, fptr);
}

int kvz_cuda_overlay_install(const char *only)
{
  if (!kvz_cuda_available()) { fprintf(stderr, "kvz-cuda overlay: %s\n", kvz_cuda_last_error()); return -1; }
  overlay_count = 0;
  overlay_filter = only;
  kvz_cuda_set_register_fn(overlay_register);
  int ok = 1;
  ok &= kvz_strategy_register_picture_cuda(NULL, KVZ_BIT_DEPTH);
  ok &= kvz_strategy_register_nal_cuda(NULL, KVZ_BIT_DEPTH);
  ok &= kvz_strategy_register_dct_cuda(NULL, KVZ_BIT_DEPTH);
  ok &= kvz_strategy_register_intra_cuda(NULL, KVZ_BIT_DEPTH);
  ok &= kvz_strategy_register_quant_plain_cuda(NULL, KVZ_BIT_DEPTH);
  for (unsigned i = 0; i < sizeof(glue_entries) / sizeof(glue_entries[0]); ++i)
    ok &= overlay_cb(NULL, glue_entries[i].type, "cuda", KVZ_CUDA_PRIORITY, glue_entries[i].fptr);
  kvz_cuda_set_register_fn(NULL);
  return ok ? overlay_count : -1;
}
