/*
 * kvz_stream_bench.c -- encoded frames/s through the UNCHANGED public libkvazaar API (kvz_api_get / config_parse /
 * encoder_open / encoder_encode, ref: src/kvazaar.h:664-829), pictures in host memory, bitstream kept.
 *
 * The same source is linked twice (integration/Makefile):
 *     kvz_stream_bench_ref   against libkvazaar_ref.so   -- the unmodified reference (its AVX2 strategies, all threads)
 *     kvz_stream_bench_ctu   against libkvazaar_ctu.so   -- the same reference with the CTU-job hooks
 *                                                          (integration/kvz_ctu_hooks.c); KVZ_CTU_PROVIDER selects
 *                                                          libkvzcuda.so
 * so both arms of bench.py measure the same loop, the one src/encmain.c:551-745 runs minus the file reader thread.
 * Built against the 10-bit reference (KVZ_BIT_DEPTH=10: kvz_stream_bench_{ref,ctu}_10b) the clip holds 16-bit
 * little-endian samples, kvz_pixel as the reference's own reader takes them.
 *
 *   kvz_stream_bench clip.yuv WxH out.hevc frames_per_step steps warmup cooldown [key=value ...]   (keys as in kvazaar --help)
 *
 * The clip's pictures are loaded before the clock starts and cycled.  (warmup + steps) * frames_per_step + cooldown
 * pictures go through ONE encoder; a step ends when the bitstream of its last picture has been returned, i.e. the steps
 * are timed output to output: with warm-up steps the clock starts when the last warm-up picture's bitstream is out
 * (without: when the first picture is handed in).  `cooldown` untimed pictures follow the timed ones so that the
 * encoder's pipeline (owf + 1 pictures in flight) is still full while the last timed step runs; cooldown = 0 puts the
 * pipeline drain inside the last step.  All pictures are written to out.hevc.  One JSON line on stdout.
 */
#define _POSIX_C_SOURCE 200809L
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>
#include <unistd.h>

#include "kvazaar.h"

static double now(void)
{
  struct timespec ts;
  clock_gettime(CLOCK_MONOTONIC, &ts);
  return ts.tv_sec + ts.tv_nsec * 1e-9;
}

int main(int argc, char **argv)
{
  if (argc < 8) { fprintf(stderr, "usage: %s clip.yuv WxH out.hevc frames_per_step steps warmup cooldown [key=value ...]\n", argv[0]); return 2; }
  const char *in = argv[1], *res = argv[2], *out = argv[3];
  const int fps_step = atoi(argv[4]), steps = atoi(argv[5]), warmup = atoi(argv[6]), cooldown = atoi(argv[7]);
  int w = 0, h = 0;
  if (sscanf(res, "%dx%d", &w, &h) != 2 || fps_step < 1 || steps < 1 || warmup < 0 || cooldown < 0) { fprintf(stderr, "bad arguments\n"); return 2; }

  const kvz_api *api = kvz_api_get(KVZ_BIT_DEPTH);
  kvz_config *cfg = api->config_alloc();
  api->config_init(cfg);
  char num[32];
  snprintf(num, sizeof(num), "%d", w); api->config_parse(cfg, "width", num);
  snprintf(num, sizeof(num), "%d", h); api->config_parse(cfg, "height", num);
  for (int i = 8; i < argc; ++i) {
    char *eq = strchr(argv[i], '=');
    if (!eq) { fprintf(stderr, "expected key=value, got %s\n", argv[i]); return 2; }
    *eq = 0;
    if (!api->config_parse(cfg, argv[i], eq + 1)) { fprintf(stderr, "config_parse(%s, %s) failed\n", argv[i], eq + 1); return 2; }
  }
  cfg->enable_logging_output = 0;

  /* the clip, resident in host memory */
  FILE *fi = fopen(in, "rb");
  if (!fi) { fprintf(stderr, "cannot open %s\n", in); return 1; }
  const size_t ysz = (size_t)w * h, csz = ysz / 4, fsz = (ysz + 2 * csz) * sizeof(kvz_pixel);    /* samples, samples, bytes */
  fseek(fi, 0, SEEK_END);
  const long clip_frames = ftell(fi) / (long)fsz;
  fseek(fi, 0, SEEK_SET);
  if (clip_frames < 1) { fprintf(stderr, "clip shorter than one picture\n"); return 1; }
  unsigned char *clip = malloc((size_t)clip_frames * fsz);
  if (!clip || fread(clip, fsz, (size_t)clip_frames, fi) != (size_t)clip_frames) { fprintf(stderr, "cannot read the clip\n"); return 1; }
  fclose(fi);

  kvz_encoder *enc = api->encoder_open(cfg);
  if (!enc) { fprintf(stderr, "encoder_open failed\n"); return 1; }
  FILE *fo = fopen(out, "wb");
  if (!fo) { fprintf(stderr, "cannot open %s\n", out); return 1; }

  const long timed_end = (long)(warmup + steps) * fps_step, total = timed_end + cooldown, first_timed = (long)warmup * fps_step;
  long fed = 0, got = 0;
  unsigned long long bytes = 0;
  double t_start = 0, t_prev = 0, *step_s = calloc((size_t)steps, sizeof(double));
  for (;;) {
    kvz_picture *pic = NULL;
    if (fed < total) {
      pic = api->picture_alloc(w, h);
      const kvz_pixel *f = (const kvz_pixel *)(clip + (size_t)(fed % clip_frames) * fsz);
      for (int r = 0; r < h; ++r) memcpy(pic->y + (size_t)r * pic->stride, f + (size_t)r * w, (size_t)w * sizeof(kvz_pixel));
      for (int r = 0; r < h / 2; ++r) {
        memcpy(pic->u + (size_t)r * (pic->stride / 2), f + ysz + (size_t)r * (w / 2), (size_t)w / 2 * sizeof(kvz_pixel));
        memcpy(pic->v + (size_t)r * (pic->stride / 2), f + ysz + csz + (size_t)r * (w / 2), (size_t)w / 2 * sizeof(kvz_pixel));
      }
      if (fed == 0 && first_timed == 0) t_start = t_prev = now();
      ++fed;
    }
    kvz_data_chunk *chunks = NULL;
    uint32_t len = 0;
    kvz_picture *rec = NULL;
    kvz_frame_info info;
    if (!api->encoder_encode(enc, pic, &chunks, &len, &rec, NULL, &info)) { fprintf(stderr, "encode failed\n"); return 1; }
    const int flushing = pic == NULL;
    if (pic) api->picture_free(pic);
    if (chunks) {
      for (kvz_data_chunk *c = chunks; c; c = c->next) { fwrite(c->data, 1, c->len, fo); bytes += c->len; }
      api->chunk_free(chunks);
      ++got;
      if (got == first_timed) t_start = t_prev = now();          /* the last warm-up picture is out */
      if (got > first_timed && got <= timed_end && (got - first_timed) % fps_step == 0) {
        const double t = now();
        step_s[(got - first_timed) / fps_step - 1] = t - t_prev;
        t_prev = t;
      }
    }
    if (rec) api->picture_free(rec);
    if (flushing && !chunks) break;        /* no more input and no more output (src/encmain.c:735) */
  }
  const double t_end = now();
  (void)t_end;
  fclose(fo);
  if (got != total) { fprintf(stderr, "expected %ld pictures out, got %ld\n", total, got); return 1; }
  double timed = 0;
  for (int i = 0; i < steps; ++i) timed += step_s[i];
  printf("{\"frames\": %ld, \"seconds\": %.6f, \"fps\": %.4f, \"frames_per_step\": %d, \"steps\": %d, \"warmup\": %d, \"cooldown\": %d, \"bytes\": %llu, \"step_seconds\": [",
         (long)steps * fps_step, timed, (double)steps * fps_step / timed, fps_step, steps, warmup, cooldown, bytes);
  for (int i = 0; i < steps; ++i) printf("%s%.6f", i ? ", " : "", step_s[i]);
  printf("]}\n");
  fflush(stdout);
  /* skip encoder_close: the provider library may be unloading its CUDA context at the same time; the OS reclaims */
  _exit(0);
}
