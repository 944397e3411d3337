/*
 * kvz_cuda_ctu.h -- C ABI of the device-resident CTU search driver (SURVEY.md §8f rank 2, VERDICT r1 item 1).
 *
 * Replaces, for all-intra pictures, the per-CTU work of the reference's CTU job
 * (encoder_state_worker_encode_lcu, src/encoderstate.c:636-773) up to the point where the bits are
 * written:
 *     kvz_search_lcu            src/search.c:1209-1250        (mode decision, reconstruction, coefficients)
 *     kvz_filter_deblock_lcu    src/filter.c:783-792
 *     kvz_sao_search_lcu        src/sao.c:671-735
 *     kvz_sao_reconstruct       src/sao.c:302-361             (final picture)
 * A whole picture is submitted; the device walks its CTUs in wavefront order (WPP dependencies, tracking the real
 * coder's CABAC context models as the host will evolve them) and returns, per CTU, exactly what the host's
 * unmodified kvz_encode_coding_tree / encode_sao need: cu_info fields, quantised coefficients, SAO parameters, plus
 * the final reconstructed picture (picture hash SEI, PSNR, --output-recon).  CABAC and the bitstream stay on the
 * host.  The binding that feeds these results into the reference is integration/kvz_ctu_hooks.c.
 *
 * Plain pointers and sizes only; no CUDA or torch types.  Result buffers are pinned host memory owned by the
 * library, valid from kvz_cuda_ctu_wait until kvz_cuda_ctu_release.
 *
 * Bit depth: kvz_cuda_ctu_config.bitdepth selects the sample type of every picture buffer crossing this interface --
 * 0 or 8: uint8_t samples, 10: uint16_t samples (kvz_pixel of a KVZ_BIT_DEPTH=10 build of the reference, values
 * 0..1023).  Strides and plane widths count samples, not bytes.  The result pointers are `const void *` to samples
 * of that type.  The source pointers of kvz_cuda_ctu_submit / _submit_device keep their `const uint8_t *` type, so
 * that providers and callers written for 8 bits build unchanged: at 10 bits the caller passes its uint16_t planes
 * cast to `const uint8_t *`, and the provider reads uint16_t samples from them.
 */
#ifndef KVZ_CUDA_CTU_H_
#define KVZ_CUDA_CTU_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* encoder configuration the intra search reads (kvz_config / encoder_control_t, see csrc/ctu/ctu_common.h) */
typedef struct kvz_cuda_ctu_config {
  int32_t width, height;            /* luma, multiples of 8 (encoder_control->in.width/height) */
  int32_t qp;                       /* fixed QP (state->qp) */
  int32_t rdo;                      /* cfg.rdo, 0..3 */
  int32_t pu_depth_intra_min, pu_depth_intra_max;
  int32_t rdoq_enable, rdoq_skip, signhide_enable, trskip_enable;
  int32_t sao_type;                 /* 0 off, 1 edge, 2 band, 3 full */
  int32_t deblock_enable, deblock_beta, deblock_tc;
  int32_t cu_split_termination;     /* 0 zero, 1 off */
  int32_t intra_rdo_et, combine_intra_cus, intra_chroma_search, full_intra_search;
  int32_t wpp;
  int32_t bitdepth;                 /* 0 or 8: 8-bit (uint8_t samples), 10: 10-bit (uint16_t samples); others are rejected */
  double  lambda, lambda_sqrt;      /* state->lambda, state->lambda_sqrt */
} kvz_cuda_ctu_config;

/* the fields of cu_info_t (src/cu.h:126-165) of an intra CU, one record per 4x4 luma block */
typedef struct kvz_cuda_ctu_cu {
  uint8_t type, depth, part_size, tr_depth;
  uint8_t tr_skip, qp;
  int8_t  mode, mode_chroma;
  uint16_t cbf;
  uint16_t pad;
} kvz_cuda_ctu_cu;

/* sao_info_t (src/sao.h:55-63) */
typedef struct kvz_cuda_ctu_sao {
  int32_t type, eo_class, ddistortion, merge_left_flag, merge_up_flag;
  int32_t band_position[2];
  int32_t offsets[10];
} kvz_cuda_ctu_sao;

typedef struct kvz_cuda_ctu_result {
  const kvz_cuda_ctu_cu *cu;        /* [(height/4) rows][cu_stride] */
  int32_t cu_stride;
  int32_t width_in_lcu, height_in_lcu;
  int32_t pad;
  const int16_t *coeff;             /* per CTU (raster): y[64*64] u[32*32] v[32*32], TUs in z-order (lcu_coeff_t, src/cu.h:292-296) */
  const kvz_cuda_ctu_sao *sao;      /* per CTU: [0] luma, [1] chroma */
  const void *rec_y, *rec_u, *rec_v;      /* final picture, stride = width (/2) samples of the configured type */
  const uint8_t *dbg_ctx;           /* per CTU: the 184 context-model bytes the CTU's search started from (may be NULL) */
  const void *dbg_y, *dbg_u, *dbg_v;      /* the search's reconstruction before deblocking (may be NULL; verification) */
} kvz_cuda_ctu_result;

typedef struct kvz_cuda_ctu_enc kvz_cuda_ctu_enc;

/* 0 if the configuration is inside the driver's scope (8- or 10-bit 4:2:0 all-intra, see csrc/ctu/ctu_search.h) */
int kvz_cuda_ctu_config_supported(const kvz_cuda_ctu_config *cfg);
/* slots = pictures that may be in flight at once (submitted, not yet released).  NULL on failure (kvz_cuda_last_error). */
kvz_cuda_ctu_enc *kvz_cuda_ctu_open(const kvz_cuda_ctu_config *cfg, int slots);
void kvz_cuda_ctu_close(kvz_cuda_ctu_enc *enc);
/* Starts the picture; returns a slot id >= 0 or a negative error.  Blocks while all slots are busy.  ctx_init: the
 * 184 CABAC context-model bytes at the start of the slice (image of cabac_data_t.ctx after kvz_init_contexts). */
int kvz_cuda_ctu_submit(kvz_cuda_ctu_enc *enc, const uint8_t *y, const uint8_t *u, const uint8_t *v, int stride_y, int stride_c,
                        const uint8_t *ctx_init, double lambda, double lambda_sqrt, int qp);
int kvz_cuda_ctu_wait(kvz_cuda_ctu_enc *enc, int slot, kvz_cuda_ctu_result *out);

/* The same with the picture already resident in device memory and the results left there (bench.py's kernel-side
 * figure; a caller that keeps the CABAC stage on the device would use it too).  Pointers of the result are device
 * pointers, valid until kvz_cuda_ctu_release. */
typedef struct kvz_cuda_ctu_device_result {
  const kvz_cuda_ctu_cu *cu;
  const int16_t *coeff;
  const kvz_cuda_ctu_sao *sao;
  const void *rec;                  /* final picture: Y, U, V planes back to back, stride = width (/2) samples */
  int32_t cu_stride, width_in_lcu, height_in_lcu;
  float search_kernel_ms;           /* device time of the picture's search launch, from the device's global timer */
} kvz_cuda_ctu_device_result;
int kvz_cuda_ctu_submit_device(kvz_cuda_ctu_enc *enc, const uint8_t *d_y, const uint8_t *d_u, const uint8_t *d_v, int stride_y, int stride_c,
                               const uint8_t *ctx_init, double lambda, double lambda_sqrt, int qp);
int kvz_cuda_ctu_wait_device(kvz_cuda_ctu_enc *enc, int slot, kvz_cuda_ctu_device_result *out);
void kvz_cuda_ctu_release(kvz_cuda_ctu_enc *enc, int slot);
/* kernels launched by this encoder so far */
uint64_t kvz_cuda_ctu_launches(const kvz_cuda_ctu_enc *enc);

#ifdef __cplusplus
}
#endif
#endif
