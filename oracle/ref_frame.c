/*
 * ref_frame.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * The back half of the reference's own CTU job (encoder_state_worker_encode_lcu: recdata to the border buffers,
 * kvz_filter_deblock_lcu, kvz_sao_search_lcu, encoder_sao_reconstruct, encode_sao + kvz_encode_coding_tree on the real
 * coder's models, the WPP hand-off) on INJECTED CTU decisions: the checker of tests/test_ctu_frame_stage.py.
 *
 * oracle/Makefile links the reference's unmodified library objects with this file and
 *   -Wl,--wrap=kvz_search_lcu          the "search" writes the case's CU records, pre-deblock reconstruction and
 *                                      coefficients where the real search leaves them (as integration/kvz_ctu_hooks.c
 *                                      does with the CTU search driver's results), and records the models the CTU
 *                                      starts from, lambda and QP; optionally it sets lambda to the case's value;
 *   -Wl,--wrap=kvz_encode_coding_tree  after the CTU's syntax (depth 0): the models and the CTU's SAO parameters;
 *   -Wl,--wrap=kvz_sao_reconstruct     the deblocked samples SAO is applied to.
 * One picture per call, through an encoder of its own opened with the case's configuration.  No arithmetic of its own.
 */
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include "global.h"
#include "kvazaar.h"
#include "kvazaar_internal.h"
#include "encoder.h"
#include "encoderstate.h"
#include "encode_coding_tree.h"
#include "cu.h"
#include "sao.h"
#include "search.h"
#include "videoframe.h"
#include "kvz_cuda_ctu.h"

void __real_kvz_search_lcu(encoder_state_t *state, int x, int y, const yuv_t *hor_buf, const yuv_t *ver_buf);
void __real_kvz_encode_coding_tree(encoder_state_t *const state, uint16_t x, uint16_t y, uint8_t depth);
void __real_kvz_sao_reconstruct(const encoder_state_t *state, const kvz_pixel *buffer, int stride, int frame_x, int frame_y,
                                int width, int height, const sao_info_t *sao, color_t color);

_Static_assert(sizeof(sao_info_t) == sizeof(kvz_cuda_ctu_sao), "sao_info_t image");
_Static_assert(sizeof(((cabac_data_t *)0)->ctx) == 184, "cabac context image");

/* the picture being encoded: inputs and capture buffers of kvzref_frame_run */
typedef struct {
  int width, height, wl;
  double lambda;
  const kvz_pixel *rec;               /* pre-deblock reconstruction: Y, U, V planes back to back, stride = width (/2) */
  const kvz_cuda_ctu_cu *cu;          /* [height / 4][width / 4] */
  const int16_t *coeff;               /* per CTU (raster): y[4096] u[1024] v[1024], lcu_coeff_t layout */
  kvz_pixel *dbk;                     /* deblocked picture (planes as rec) */
  kvz_cuda_ctu_sao *sao;              /* per CTU: [0] luma, [1] chroma */
  uint8_t *ctx_start, *ctx_end;       /* per CTU: 184 model bytes */
  double *lam;                        /* per CTU: lambda, lambda_sqrt */
  int32_t *qp;                        /* per CTU */
  int32_t *visits;                    /* per CTU: searched, syntax written */
} run_t;

static run_t *g_run;

static void cu_from_rec(cu_info_t *to, const kvz_cuda_ctu_cu *r)
{
  memset(to, 0, sizeof(*to));
  to->type = r->type; to->depth = r->depth; to->part_size = r->part_size; to->tr_depth = r->tr_depth;
  to->tr_skip = r->tr_skip; to->cbf = r->cbf; to->qp = r->qp;
  to->intra.mode = r->mode; to->intra.mode_chroma = r->mode_chroma;
}

void __wrap_kvz_search_lcu(encoder_state_t *state, int x, int y, const yuv_t *hor_buf, const yuv_t *ver_buf)
{
  run_t *r = g_run;
  if (!r) { __real_kvz_search_lcu(state, x, y, hor_buf, ver_buf); return; }
  videoframe_t *frame = state->tile->frame;
  const int lcu = (y / 64) * r->wl + x / 64;
  memcpy(r->ctx_start + (size_t)lcu * 184, &state->cabac.ctx, 184);
  /* the search starts from the coder's models (search.c kvz_search_lcu) and never adapts the SAO models, which
   * kvz_sao_search_lcu reads from state->search_cabac afterwards */
  memcpy(&state->search_cabac, &state->cabac, sizeof(cabac_data_t));
  state->search_cabac.only_count = 1;
  if (r->lambda > 0) { state->lambda = r->lambda; state->lambda_sqrt = sqrt(r->lambda); }
  r->lam[2 * lcu] = state->lambda; r->lam[2 * lcu + 1] = state->lambda_sqrt;
  r->qp[lcu] = state->qp;
  r->visits[2 * lcu] += 1;
  const int W = r->width, H = r->height, Wc = W / 2, Hc = H / 2;
  const int x_max = MIN(x + 64, W) - x, y_max = MIN(y + 64, H) - y;
  for (int sy = 0; sy < y_max; sy += 4)
    for (int sx = 0; sx < x_max; sx += 4)
      cu_from_rec(kvz_cu_array_at(frame->cu_array, x + sx, y + sy), &r->cu[((y + sy) >> 2) * (W / 4) + ((x + sx) >> 2)]);
  const int16_t *co = r->coeff + (size_t)lcu * 6144;
  memcpy(state->coeff->y, co, 4096 * sizeof(int16_t));
  memcpy(state->coeff->u, co + 4096, 1024 * sizeof(int16_t));
  memcpy(state->coeff->v, co + 5120, 1024 * sizeof(int16_t));
  kvz_picture *rec = frame->rec;
  const kvz_pixel *ry = r->rec, *ru = ry + (size_t)W * H, *rv = ru + (size_t)Wc * Hc;
  for (int yy = 0; yy < y_max; ++yy) memcpy(rec->y + (size_t)(y + yy) * rec->stride + x, ry + (size_t)(y + yy) * W + x, x_max * sizeof(kvz_pixel));
  for (int yy = 0; yy < y_max / 2; ++yy) {
    memcpy(rec->u + (size_t)(y / 2 + yy) * (rec->stride / 2) + x / 2, ru + (size_t)(y / 2 + yy) * Wc + x / 2, x_max / 2 * sizeof(kvz_pixel));
    memcpy(rec->v + (size_t)(y / 2 + yy) * (rec->stride / 2) + x / 2, rv + (size_t)(y / 2 + yy) * Wc + x / 2, x_max / 2 * sizeof(kvz_pixel));
  }
}

void __wrap_kvz_encode_coding_tree(encoder_state_t *const state, uint16_t x, uint16_t y, uint8_t depth)
{
  __real_kvz_encode_coding_tree(state, x, y, depth);
  run_t *r = g_run;
  if (!r || depth != 0) return;
  const videoframe_t *frame = state->tile->frame;
  const int lcu = (y / 64) * r->wl + x / 64;
  memcpy(r->ctx_end + (size_t)lcu * 184, &state->cabac.ctx, 184);
  if (state->encoder_control->cfg.sao_type) {
    memcpy(&r->sao[2 * lcu], &frame->sao_luma[lcu], sizeof(sao_info_t));
    memcpy(&r->sao[2 * lcu + 1], &frame->sao_chroma[lcu], sizeof(sao_info_t));
  }
  r->visits[2 * lcu + 1] += 1;
}

/* the buffer holds the deblocked samples of the area (encoder_sao_reconstruct copies them before SAO changes the
 * picture); every sample of the picture passes through here exactly once */
void __wrap_kvz_sao_reconstruct(const encoder_state_t *state, const kvz_pixel *buffer, int stride, int frame_x, int frame_y,
                                int width, int height, const sao_info_t *sao, color_t color)
{
  run_t *r = g_run;
  if (r) {
    const int W = r->width, H = r->height;
    const int pw = color == COLOR_Y ? W : W / 2;
    kvz_pixel *p = r->dbk + (color == COLOR_Y ? 0 : (size_t)W * H + (color == COLOR_V ? (size_t)(W / 2) * (H / 2) : 0));
    for (int yy = 0; yy < height; ++yy) memcpy(p + (size_t)(frame_y + yy) * pw + frame_x, buffer + (size_t)yy * stride, width * sizeof(kvz_pixel));
  }
  __real_kvz_sao_reconstruct(state, buffer, stride, frame_x, frame_y, width, height, sao, color);
}

/* One all-intra picture (intra period 1, WPP, no threads, no OWF, fixed QP) whose every CTU takes the injected decisions.
 * sao_type: 0 off, 1 edge, 2 band, 3 both.  lambda > 0 replaces state->lambda (and lambda_sqrt) in every CTU.
 * src / rec: Y, U, V planes back to back, stride = width (/2).  Outputs: the deblocked picture (with SAO off: the final
 * picture), the final picture, per CTU both SAO records (SAO on only), the 184 model bytes at the CTU's start and after
 * its syntax, lambda / lambda_sqrt, QP, and how often the CTU was searched / coded ([nctu][2]).
 * Returns 0, or -1 when the encoder refuses the configuration or produces no picture. */
int kvzref_frame_run(int width, int height, int qp, int sao_type, int deblock, int beta, int tc, int trskip, double lambda,
                     const kvz_pixel *src, const kvz_pixel *rec, const kvz_cuda_ctu_cu *cu, const int16_t *coeff,
                     kvz_pixel *dbk, kvz_pixel *out, kvz_cuda_ctu_sao *sao, uint8_t *ctx_start, uint8_t *ctx_end,
                     double *lam, int32_t *qp_out, int32_t *visits)
{
  const kvz_api *api = kvz_api_get(KVZ_BIT_DEPTH);
  kvz_config *cfg = api->config_alloc();
  if (!cfg) return -1;
  api->config_init(cfg);
  cfg->width = width; cfg->height = height; cfg->qp = qp;
  cfg->intra_period = 1; cfg->gop_len = 0;
  cfg->wpp = 1; cfg->threads = 0; cfg->owf = 0;
  cfg->hash = KVZ_HASH_NONE; cfg->enable_logging_output = 0;
  cfg->input_bitdepth = KVZ_BIT_DEPTH;
  cfg->sao_type = sao_type;
  cfg->deblock_enable = deblock; cfg->deblock_beta = beta; cfg->deblock_tc = tc;
  cfg->trskip_enable = trskip; cfg->signhide_enable = 0;
  kvz_encoder *enc = api->encoder_open(cfg);
  if (!enc) { api->config_destroy(cfg); return -1; }
  const int wl = (width + 63) / 64;
  run_t r = { width, height, wl, lambda, rec, cu, coeff, dbk, sao, ctx_start, ctx_end, lam, qp_out, visits };
  kvz_picture *in = api->picture_alloc(width, height);
  const size_t ny = (size_t)width * height, nc = ny / 4;
  for (int y = 0; y < height; ++y) memcpy(in->y + (size_t)y * in->stride, src + (size_t)y * width, width * sizeof(kvz_pixel));
  for (int y = 0; y < height / 2; ++y) {
    memcpy(in->u + (size_t)y * (in->stride / 2), src + ny + (size_t)y * (width / 2), width / 2 * sizeof(kvz_pixel));
    memcpy(in->v + (size_t)y * (in->stride / 2), src + ny + nc + (size_t)y * (width / 2), width / 2 * sizeof(kvz_pixel));
  }
  g_run = &r;
  kvz_picture *pic = NULL;
  kvz_data_chunk *data = NULL;
  uint32_t len = 0;
  int ok = api->encoder_encode(enc, in, &data, &len, &pic, NULL, NULL);
  for (int i = 0; ok && !pic && i < 4; ++i) {
    if (data) { api->chunk_free(data); data = NULL; }
    ok = api->encoder_encode(enc, NULL, &data, &len, &pic, NULL, NULL);
  }
  g_run = NULL;
  int rc = -1;
  if (ok && pic) {
    for (int y = 0; y < height; ++y) memcpy(out + (size_t)y * width, pic->y + (size_t)y * pic->stride, width * sizeof(kvz_pixel));
    for (int y = 0; y < height / 2; ++y) {
      memcpy(out + ny + (size_t)y * (width / 2), pic->u + (size_t)y * (pic->stride / 2), width / 2 * sizeof(kvz_pixel));
      memcpy(out + ny + nc + (size_t)y * (width / 2), pic->v + (size_t)y * (pic->stride / 2), width / 2 * sizeof(kvz_pixel));
    }
    if (!sao_type) memcpy(dbk, out, (ny + 2 * nc) * sizeof(kvz_pixel));
    rc = 0;
  }
  if (data) api->chunk_free(data);
  api->picture_free(pic);
  api->picture_free(in);
  api->encoder_close(enc);
  api->config_destroy(cfg);
  return rc;
}
