/*
 * kvz_ctu_hooks.c -- binds the CTU search driver (include/kvz_cuda_ctu.h) into the UNMODIFIED reference encoder.
 *
 * The four functions of the CTU job that the driver replaces are intercepted at link time
 * (-Wl,--wrap=..., see oracle/Makefile "ctu"); the reference sources are compiled as they are:
 *     kvz_search_lcu           (called at src/encoderstate.c:660)
 *     kvz_filter_deblock_lcu   (src/encoderstate.c:671)
 *     kvz_sao_search_lcu       (src/encoderstate.c:682)
 *     kvz_sao_reconstruct      (src/encoderstate.c:351, inside encoder_sao_reconstruct)
 * A maintainer integrating the driver would put the same four `if (driver active)` branches at those call sites
 * (INTEGRATION.md).  Everything else -- threading, WPP jobs, kvz_encode_coding_tree, encode_sao, CABAC, NAL writing,
 * picture hash -- is the reference's own code running on the driver's results.
 *
 * Environment:
 *   KVZ_CTU_PROVIDER = path of a library exporting the kvz_cuda_ctu_* ABI (libkvzcuda.so; tests: the host build)
 *   KVZ_CTU_MODE     = replace (default) | verify  (verify: the reference searches too, differences are reported)
 *   KVZ_CTU_SLOTS    = picture slots of the provider (default and minimum: owf + 1, the pictures the encoder keeps in
 *                      flight -- a worker blocked on a busy slot could otherwise starve the pictures that hold the slots)
 * Without KVZ_CTU_PROVIDER, or when the configuration is outside the driver's scope, every hook falls through.
 * The same source serves the 8-bit and the 10-bit build of the reference (KVZ_BIT_DEPTH): pictures cross the driver's
 * interface as kvz_pixel samples, and kvz_cuda_ctu_config.bitdepth tells the provider which.
 */
#define _GNU_SOURCE
#include <dlfcn.h>
#include <pthread.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "encoderstate.h"
#include "encoder.h"
#include "search.h"
#include "filter.h"
#include "sao.h"
#include "videoframe.h"
#include "cu.h"
#include "kvz_cuda_ctu.h"

void __real_kvz_search_lcu(encoder_state_t *state, int x, int y, const yuv_t *hor_buf, const yuv_t *ver_buf);
void __real_kvz_filter_deblock_lcu(encoder_state_t *state, int x_px, int y_px);
void __real_kvz_sao_search_lcu(const encoder_state_t *state, int lcu_x, int lcu_y);
void __real_kvz_sao_reconstruct(const encoder_state_t *state, const kvz_pixel *buffer, int stride, int frame_x, int frame_y,
                                int width, int height, const sao_info_t *sao, color_t color);

typedef struct {
  void *lib;
  int (*supported)(const kvz_cuda_ctu_config *);
  kvz_cuda_ctu_enc *(*open)(const kvz_cuda_ctu_config *, int);
  void (*close)(kvz_cuda_ctu_enc *);
  int (*submit)(kvz_cuda_ctu_enc *, const uint8_t *, const uint8_t *, const uint8_t *, int, int, const uint8_t *, double, double, int);
  int (*wait)(kvz_cuda_ctu_enc *, int, kvz_cuda_ctu_result *);
  void (*release)(kvz_cuda_ctu_enc *, int);
} provider_t;

typedef struct {
  const videoframe_t *frame;     /* key */
  int slot;
  int lcus_left;
  kvz_cuda_ctu_result res;
} job_t;

#define MAX_JOBS 512
static provider_t g_prov;
static kvz_cuda_ctu_enc *g_enc;
static const encoder_control_t *g_ctrl;
static int g_state;            /* 0 unknown, 1 active, -1 inactive */
static int g_verify;
static long g_mismatch;
static job_t g_jobs[MAX_JOBS];
static pthread_mutex_t g_lock = PTHREAD_MUTEX_INITIALIZER;

static void fill_config(const encoder_state_t *state, kvz_cuda_ctu_config *c)
{
  const encoder_control_t *ctrl = state->encoder_control;
  const kvz_config *cfg = &ctrl->cfg;
  memset(c, 0, sizeof(*c));
  c->width = state->tile->frame->width; c->height = state->tile->frame->height;
  c->qp = state->qp;
  c->rdo = cfg->rdo;
  c->pu_depth_intra_min = cfg->pu_depth_intra.min[0]; c->pu_depth_intra_max = cfg->pu_depth_intra.max[0];
  c->rdoq_enable = cfg->rdoq_enable; c->rdoq_skip = cfg->rdoq_skip;
  c->signhide_enable = cfg->signhide_enable; c->trskip_enable = cfg->trskip_enable;
  c->sao_type = cfg->sao_type;
  c->deblock_enable = cfg->deblock_enable; c->deblock_beta = cfg->deblock_beta; c->deblock_tc = cfg->deblock_tc;
  c->cu_split_termination = cfg->cu_split_termination == KVZ_CU_SPLIT_TERMINATION_OFF;
  c->intra_rdo_et = cfg->intra_rdo_et; c->combine_intra_cus = cfg->combine_intra_cus;
  c->intra_chroma_search = cfg->intra_chroma_search; c->full_intra_search = cfg->full_intra_search;
  c->wpp = cfg->wpp;
  c->bitdepth = ctrl->bitdepth;
  c->lambda = state->lambda; c->lambda_sqrt = state->lambda_sqrt;
}

static int cfg_owf(const encoder_state_t *state) { return state->encoder_control->cfg.owf > 0 ? state->encoder_control->cfg.owf : 0; }

/* is this encoder inside the driver's scope?  (ctu_search.h header) */
static int config_in_scope(const encoder_state_t *state)
{
  const encoder_control_t *ctrl = state->encoder_control;
  const kvz_config *cfg = &ctrl->cfg;
  if (ctrl->bitdepth != KVZ_BIT_DEPTH || (ctrl->bitdepth != 8 && ctrl->bitdepth != 10) || ctrl->chroma_format != KVZ_CSP_420) return 0;
  if (cfg->intra_period != 1) return 0;
  if (cfg->lossless || cfg->tr_depth_intra != 0 || cfg->rdo > 3) return 0;
  if (ctrl->scaling_list.enable) return 0;
  if (cfg->tiles_width_count != 1 || cfg->tiles_height_count != 1 || cfg->slices) return 0;
  if (!cfg->wpp) return 0;
  if (cfg->target_bitrate > 0 || cfg->roi.file_path || cfg->vaq || cfg->set_qp_in_cu || state->frame->max_qp_delta_depth >= 0) return 0;
  if (cfg->crypto_features || cfg->implicit_rdpcm || cfg->ml_pu_depth_intra) return 0;
  if (state->qp < cfg->fast_residual_cost_limit && state->qp < MAX_FAST_COEFF_COST_QP) return 0;
  if (cfg->pu_depth_intra.min[0] < 1) return 0;
  for (int i = 1; i < KVZ_MAX_GOP_LAYERS; ++i) if (cfg->pu_depth_intra.min[i] >= 0 || cfg->pu_depth_intra.max[i] >= 0) return 0;
  if (state->constraint && ((constraint_t *)state->constraint)->ml_intra_depth_ctu) return 0;
  return 1;
}

static int driver_active(const encoder_state_t *state)
{
  if (__atomic_load_n(&g_state, __ATOMIC_ACQUIRE)) return g_state > 0 && state->encoder_control == g_ctrl && state->frame->slicetype == KVZ_SLICE_I;
  pthread_mutex_lock(&g_lock);
  if (!g_state) {
    int st = -1;             /* published only when the set-up is complete: other workers wait on the lock */
    const char *path = getenv("KVZ_CTU_PROVIDER");
    if (path && *path && config_in_scope(state)) {
      g_prov.lib = dlopen(path, RTLD_NOW | RTLD_LOCAL);
      if (!g_prov.lib) fprintf(stderr, "kvz-ctu: cannot load %s: %s\n", path, dlerror());
      else {
        g_prov.supported = dlsym(g_prov.lib, "kvz_cuda_ctu_config_supported");
        g_prov.open = dlsym(g_prov.lib, "kvz_cuda_ctu_open");
        g_prov.close = dlsym(g_prov.lib, "kvz_cuda_ctu_close");
        g_prov.submit = dlsym(g_prov.lib, "kvz_cuda_ctu_submit");
        g_prov.wait = dlsym(g_prov.lib, "kvz_cuda_ctu_wait");
        g_prov.release = dlsym(g_prov.lib, "kvz_cuda_ctu_release");
        kvz_cuda_ctu_config c;
        fill_config(state, &c);
        const char *slots = getenv("KVZ_CTU_SLOTS");
        const char *mode = getenv("KVZ_CTU_MODE");
        g_verify = mode && strcmp(mode, "verify") == 0;
        if (g_prov.supported && g_prov.open && g_prov.submit && g_prov.wait && g_prov.release && g_prov.supported(&c) == 0)
        {
          int n = cfg_owf(state) + 1;
          if (slots && atoi(slots) > n) n = atoi(slots);
          g_enc = g_prov.open(&c, n);
        }
        if (g_enc) { g_ctrl = state->encoder_control; st = 1; fprintf(stderr, "kvz-ctu: CTU search driver active (%s%s)\n", path, g_verify ? ", verify" : ""); }
        else fprintf(stderr, "kvz-ctu: provider refused the configuration, using the reference path\n");
      }
    }
    __atomic_store_n(&g_state, st, __ATOMIC_RELEASE);
  }
  pthread_mutex_unlock(&g_lock);
  return g_state > 0 && state->encoder_control == g_ctrl && state->frame->slicetype == KVZ_SLICE_I;
}

static job_t *job_find(const videoframe_t *frame)
{
  for (int i = 0; i < MAX_JOBS; ++i) if (g_jobs[i].frame == frame) return &g_jobs[i];
  return NULL;
}

/* the job of the picture this CTU belongs to; the first CTU of a picture (0,0) submits it and waits for the device */
static job_t *job_get(encoder_state_t *state, int x, int y)
{
  const videoframe_t *frame = state->tile->frame;
  pthread_mutex_lock(&g_lock);
  job_t *j = job_find(frame);
  if (!j && x == 0 && y == 0) {
    j = job_find(NULL);
    if (j) { j->frame = frame; j->slot = -1; j->lcus_left = frame->width_in_lcu * frame->height_in_lcu; }
  }
  pthread_mutex_unlock(&g_lock);
  if (!j) { fprintf(stderr, "kvz-ctu: no job for CTU (%d,%d)\n", x, y); abort(); }
  if (j->slot < 0) {
    /* (0,0) runs before every other CTU of the picture: no concurrent access to this job yet */
    const kvz_picture *src = frame->source;
    static _Thread_local uint8_t ctx[184];
    _Static_assert(sizeof(state->cabac.ctx) == 184, "cabac context image");
    memcpy(ctx, &state->cabac.ctx, 184);
    j->slot = g_prov.submit(g_enc, (const uint8_t *)src->y, (const uint8_t *)src->u, (const uint8_t *)src->v, src->stride, src->stride / 2, ctx, state->lambda, state->lambda_sqrt, state->qp);
    if (j->slot < 0 || g_prov.wait(g_enc, j->slot, &j->res) != 0) { fprintf(stderr, "kvz-ctu: device search failed\n"); abort(); }
    if (!g_verify) {
      kvz_picture *rec = frame->rec;
      const kvz_pixel *ry = j->res.rec_y, *ru = j->res.rec_u, *rv = j->res.rec_v;
      const size_t w = frame->width, wc = w / 2;
      for (int r = 0; r < frame->height; ++r) memcpy(rec->y + (size_t)r * rec->stride, ry + r * w, w * sizeof(kvz_pixel));
      for (int r = 0; r < frame->height / 2; ++r) {
        memcpy(rec->u + (size_t)r * (rec->stride / 2), ru + r * wc, wc * sizeof(kvz_pixel));
        memcpy(rec->v + (size_t)r * (rec->stride / 2), rv + r * wc, wc * sizeof(kvz_pixel));
      }
    }
  }
  return j;
}

static void job_done_lcu(job_t *j)
{
  pthread_mutex_lock(&g_lock);
  if (--j->lcus_left == 0) { g_prov.release(g_enc, j->slot); j->frame = NULL; }
  pthread_mutex_unlock(&g_lock);
}

static void cu_from_rec(cu_info_t *to, const kvz_cuda_ctu_cu *r)
{
  memset(to, 0, sizeof(*to));
  to->type = r->type; to->depth = r->depth; to->part_size = r->part_size; to->tr_depth = r->tr_depth;
  to->tr_skip = r->tr_skip; to->cbf = r->cbf; to->qp = r->qp;
  to->intra.mode = r->mode; to->intra.mode_chroma = r->mode_chroma;
}

static void report(const char *what, int x, int y, int sx, int sy, long a, long b)
{
  if (__sync_add_and_fetch(&g_mismatch, 1) <= 40)
    fprintf(stderr, "kvz-ctu VERIFY MISMATCH %s: CTU (%d,%d) at (%d,%d): reference %ld, driver %ld\n", what, x / 64, y / 64, sx, sy, a, b);
}

void __wrap_kvz_search_lcu(encoder_state_t *state, int x, int y, const yuv_t *hor_buf, const yuv_t *ver_buf)
{
  if (!driver_active(state)) { __real_kvz_search_lcu(state, x, y, hor_buf, ver_buf); return; }
  job_t *j = job_get(state, x, y);
  videoframe_t *frame = state->tile->frame;
  const int wl = frame->width_in_lcu, lcu = (y / 64) * wl + x / 64;
  const int16_t *co = j->res.coeff + (size_t)lcu * 6144;
  const int x_max = MIN(x + 64, frame->width) - x, y_max = MIN(y + 64, frame->height) - y;
  if (g_verify) {
    if (j->res.dbg_ctx && memcmp(j->res.dbg_ctx + (size_t)lcu * 184, &state->cabac.ctx, 184) != 0) {
      const uint8_t *a = (const uint8_t *)&state->cabac.ctx, *b = j->res.dbg_ctx + (size_t)lcu * 184;
      for (int i = 0; i < 184; ++i) if (a[i] != b[i]) { report("cabac model at CTU start", x, y, i, 0, a[i], b[i]); break; }
    }
    __real_kvz_search_lcu(state, x, y, hor_buf, ver_buf);
    for (int sy = 0; sy < y_max; sy += 4)
      for (int sx = 0; sx < x_max; sx += 4) {
        const cu_info_t *a = kvz_cu_array_at_const(frame->cu_array, x + sx, y + sy);
        const kvz_cuda_ctu_cu *b = &j->res.cu[((y + sy) >> 2) * j->res.cu_stride + ((x + sx) >> 2)];
        if (a->type != b->type) report("type", x, y, sx, sy, a->type, b->type);
        else if (a->depth != b->depth) report("depth", x, y, sx, sy, a->depth, b->depth);
        else if (a->part_size != b->part_size) report("part_size", x, y, sx, sy, a->part_size, b->part_size);
        else if (a->tr_depth != b->tr_depth) report("tr_depth", x, y, sx, sy, a->tr_depth, b->tr_depth);
        else if (a->intra.mode != b->mode) report("mode", x, y, sx, sy, a->intra.mode, b->mode);
        else if (a->intra.mode_chroma != b->mode_chroma) report("mode_chroma", x, y, sx, sy, a->intra.mode_chroma, b->mode_chroma);
        else if (a->cbf != b->cbf) report("cbf", x, y, sx, sy, a->cbf, b->cbf);
        else if (a->tr_skip != b->tr_skip) report("tr_skip", x, y, sx, sy, a->tr_skip, b->tr_skip);
      }
    if (j->res.dbg_y) {
      const kvz_picture *rec = frame->rec;
      const kvz_pixel *dy = j->res.dbg_y, *du = j->res.dbg_u, *dv = j->res.dbg_v;
      int done = 0;
      for (int yy = 0; yy < y_max && !done; ++yy)
        for (int xx = 0; xx < x_max; ++xx)
          if (rec->y[(size_t)(y + yy) * rec->stride + x + xx] != dy[(size_t)(y + yy) * frame->width + x + xx]) {
            report("rec_y (before deblocking)", x, y, xx, yy, rec->y[(size_t)(y + yy) * rec->stride + x + xx], dy[(size_t)(y + yy) * frame->width + x + xx]); done = 1; break; }
      done = 0;
      for (int yy = 0; yy < y_max / 2 && !done; ++yy)
        for (int xx = 0; xx < x_max / 2; ++xx) {
          const size_t a = (size_t)(y / 2 + yy) * (rec->stride / 2) + x / 2 + xx, b = (size_t)(y / 2 + yy) * (frame->width / 2) + x / 2 + xx;
          if (rec->u[a] != du[b]) { report("rec_u (before deblocking)", x, y, xx, yy, rec->u[a], du[b]); done = 1; break; }
          if (rec->v[a] != dv[b]) { report("rec_v (before deblocking)", x, y, xx, yy, rec->v[a], dv[b]); done = 1; break; }
        }
    }
    for (int i = 0; i < 4096; ++i) if (state->coeff->y[i] != co[i]) { report("coeff_y", x, y, i, 0, state->coeff->y[i], co[i]); break; }
    for (int i = 0; i < 1024; ++i) if (state->coeff->u[i] != co[4096 + i]) { report("coeff_u", x, y, i, 0, state->coeff->u[i], co[4096 + i]); break; }
    for (int i = 0; i < 1024; ++i) if (state->coeff->v[i] != co[5120 + i]) { report("coeff_v", x, y, i, 0, state->coeff->v[i], co[5120 + i]); break; }
    if (!state->encoder_control->cfg.sao_type) job_done_lcu(j);
    return;
  }
  for (int sy = 0; sy < y_max; sy += 4)
    for (int sx = 0; sx < x_max; sx += 4)
      cu_from_rec(kvz_cu_array_at(frame->cu_array, x + sx, y + sy), &j->res.cu[((y + sy) >> 2) * j->res.cu_stride + ((x + sx) >> 2)]);
  memcpy(state->coeff->y, co, 4096 * sizeof(int16_t));
  memcpy(state->coeff->u, co + 4096, 1024 * sizeof(int16_t));
  memcpy(state->coeff->v, co + 5120, 1024 * sizeof(int16_t));
  if (!state->encoder_control->cfg.sao_type) job_done_lcu(j);
}

void __wrap_kvz_filter_deblock_lcu(encoder_state_t *state, int x_px, int y_px)
{
  if (!driver_active(state) || g_verify) __real_kvz_filter_deblock_lcu(state, x_px, y_px);
}

void __wrap_kvz_sao_search_lcu(const encoder_state_t *state, int lcu_x, int lcu_y)
{
  if (!driver_active(state)) { __real_kvz_sao_search_lcu(state, lcu_x, lcu_y); return; }
  videoframe_t *frame = state->tile->frame;
  pthread_mutex_lock(&g_lock);
  job_t *j = job_find(frame);
  pthread_mutex_unlock(&g_lock);
  if (!j) { fprintf(stderr, "kvz-ctu: no job for SAO of CTU (%d,%d)\n", lcu_x, lcu_y); abort(); }
  const int i = lcu_y * frame->width_in_lcu + lcu_x;
  const kvz_cuda_ctu_sao *s = &j->res.sao[2 * i];
  _Static_assert(sizeof(sao_info_t) == sizeof(kvz_cuda_ctu_sao), "sao_info_t image");
  if (g_verify) {
    __real_kvz_sao_search_lcu(state, lcu_x, lcu_y);
    for (int k = 0; k < 2; ++k) {
      const sao_info_t *a = k ? &frame->sao_chroma[i] : &frame->sao_luma[i];
      const kvz_cuda_ctu_sao *b = s + k;
      if ((int)a->type != b->type) report(k ? "sao_chroma.type" : "sao_luma.type", lcu_x * 64, lcu_y * 64, 0, 0, a->type, b->type);
      else if (a->merge_left_flag != b->merge_left_flag || a->merge_up_flag != b->merge_up_flag) report("sao merge flags", lcu_x * 64, lcu_y * 64, k, 0, a->merge_left_flag * 2 + a->merge_up_flag, b->merge_left_flag * 2 + b->merge_up_flag);
      else if (a->type != SAO_TYPE_NONE) {
        if (a->type == SAO_TYPE_EDGE && (int)a->eo_class != b->eo_class) report("sao eo_class", lcu_x * 64, lcu_y * 64, k, 0, a->eo_class, b->eo_class);
        for (int o = 1; o < (k ? 10 : 5); ++o) if (o != 5 && a->offsets[o] != b->offsets[o]) { report("sao offset", lcu_x * 64, lcu_y * 64, k, o, a->offsets[o], b->offsets[o]); break; }
        if (a->type == SAO_TYPE_BAND) for (int o = 0; o < (k ? 2 : 1); ++o) if (a->band_position[o] != b->band_position[o]) report("sao band_position", lcu_x * 64, lcu_y * 64, k, o, a->band_position[o], b->band_position[o]);
      }
    }
  } else {
    memcpy(&frame->sao_luma[i], s, sizeof(sao_info_t));
    memcpy(&frame->sao_chroma[i], s + 1, sizeof(sao_info_t));
  }
  job_done_lcu(j);
}

void __wrap_kvz_sao_reconstruct(const encoder_state_t *state, const kvz_pixel *buffer, int stride, int frame_x, int frame_y,
                                int width, int height, const sao_info_t *sao, color_t color)
{
  if (!driver_active(state) || g_verify) __real_kvz_sao_reconstruct(state, buffer, stride, frame_x, frame_y, width, height, sao, color);
}

long kvz_ctu_hooks_mismatches(void) { return g_mismatch; }

__attribute__((destructor)) static void hooks_exit(void)
{
  if (g_verify) fprintf(stderr, "kvz-ctu: verify finished, %ld mismatches\n", g_mismatch);
  /* the provider library may already be tearing down at process exit: leave the encoder to the OS */
}
