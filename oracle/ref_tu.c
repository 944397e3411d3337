/*
 * ref_tu.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * One intra transform unit as the CTU search evaluates it, through the UNMODIFIED reference (linked to
 * oracle/_ref/libkvazaar_ref.so by oracle/Makefile): the checker of tests/test_ctu_tu_jobs.py.  A library of its own
 * (libkvzref_tu.so), with an encoder of its own, because every call rewrites the configuration's switches.
 * It contains no arithmetic of its own.
 */
#include <stdlib.h>
#include <string.h>

#include "global.h"
#include "kvazaar.h"
#include "kvazaar_internal.h"
#include "encoder.h"
#include "encoderstate.h"
#include "cu.h"
#include "intra.h"
#include "rdo.h"
#include "transform.h"
#include "strategies/strategies-quant.h"
#include "strategies/strategies-picture.h"

typedef struct {
  const kvz_api *api;
  kvz_config *cfg;
  kvz_encoder *enc;
} kvzref_tu_ctx;

/* opening the encoder also selects the strategies the reference CLI runs (kvazaar.c: kvz_strategyselector_init) */
kvzref_tu_ctx *kvzref_tu_open(void)
{
  kvzref_tu_ctx *c = calloc(1, sizeof(*c));
  c->api = kvz_api_get(KVZ_BIT_DEPTH);
  c->cfg = c->api->config_alloc();
  c->api->config_init(c->cfg);
  c->cfg->width = 64; c->cfg->height = 64; c->cfg->qp = 22;
  c->cfg->threads = 0; c->cfg->owf = 0; c->cfg->wpp = 0;
  c->cfg->hash = KVZ_HASH_NONE;
  c->cfg->enable_logging_output = 0;
  c->enc = c->api->encoder_open(c->cfg);
  if (!c->enc) { c->api->config_destroy(c->cfg); free(c); return NULL; }
  return c;
}

/* Prediction from unfiltered references (kvz_intra_predict), kvz_quantize_residual -- or kvz_quantize_residual_trskip
 * for a 4x4 luma unit when transform skip is enabled and alt < 0; alt 0 / 1 forces the transform / transform skip --
 * then kvz_pixels_calc_ssd and kvz_get_coeff_cost on the search models.  The CU record is intra with depth / tr_depth,
 * NxN when nxn is set.  fast_residual_cost_limit is 0 (the accurate CABAC cost).  Samples of src / pred / rec and the
 * levels are n x n with stride n.  out_i: has, tr_skip, ssd.  Returns the coefficient bits. */
double kvzref_intra_tu(kvzref_tu_ctx *c, int qp, double lambda, int rdoq, int rdoq_skip, int signhide, int trskip,
                       const uint8_t *cabac0, const uint8_t *sc, int color, int log2n, int depth, int tr_depth, int nxn,
                       int mode, int scan, int alt, const kvz_pixel *top, const kvz_pixel *left, const kvz_pixel *src,
                       kvz_pixel *pred, kvz_pixel *rec, coeff_t *coeff, int32_t *out_i)
{
  encoder_state_t *st = &c->enc->states[0];
  encoder_control_t *ctrl = (encoder_control_t *)st->encoder_control;
  ctrl->cfg.rdoq_enable = rdoq; ctrl->cfg.rdoq_skip = rdoq_skip; ctrl->cfg.signhide_enable = signhide;
  ctrl->cfg.trskip_enable = trskip; ctrl->cfg.fast_residual_cost_limit = 0;
  st->qp = (int8_t)qp;
  st->frame->slicetype = KVZ_SLICE_I;
  st->lambda = lambda;
  memcpy(&st->cabac.ctx, cabac0, sizeof(st->cabac.ctx));
  memcpy(&st->search_cabac.ctx, sc, sizeof(st->search_cabac.ctx));
  st->search_cabac.update = 0;
  cu_info_t cu; memset(&cu, 0, sizeof(cu));
  cu.type = CU_INTRA; cu.depth = depth; cu.tr_depth = tr_depth; cu.part_size = nxn ? SIZE_NxN : SIZE_2Nx2N;
  cu.intra.mode = (int8_t)mode; cu.intra.mode_chroma = (int8_t)mode;
  const int n = 1 << log2n;
  kvz_intra_references refs; memset(&refs, 0, sizeof(refs));
  memcpy(refs.ref.top, top, (2 * n + 1) * sizeof(kvz_pixel));
  memcpy(refs.ref.left, left, (2 * n + 1) * sizeof(kvz_pixel));
  refs.filtered_initialized = false;
  kvz_intra_predict(&refs, (int_fast8_t)log2n, (int_fast8_t)mode, (color_t)color, pred, color == COLOR_Y);
  int8_t ts = 0;
  int has;
  if (alt < 0 && trskip && n == 4 && color == COLOR_Y)
    has = kvz_quantize_residual_trskip(st, &cu, n, (color_t)color, (coeff_scan_order_t)scan, &ts, n, n, src, pred, rec, coeff);
  else
    has = kvz_quantize_residual(st, &cu, n, (color_t)color, (coeff_scan_order_t)scan, alt == 1, n, n, src, pred, rec, coeff, false);
  out_i[0] = has;
  out_i[1] = ts;
  out_i[2] = (int32_t)kvz_pixels_calc_ssd(src, rec, n, n, n);
  return kvz_get_coeff_cost(st, coeff, n, color == COLOR_Y ? 0 : 2, (int8_t)scan);
}
