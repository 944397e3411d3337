// ctu_hostsim_10b.cpp -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
//
// The host build of the CTU search driver (see ctu_hostsim.cpp: the single-source algorithm of csrc/ctu/*.h with a
// "CTA" of one thread behind the C ABI of include/kvz_cuda_ctu.h) with BOTH instantiations of the algorithm:
// cfg.bitdepth picks one (0 / 8: uint8_t, 10: uint16_t samples) and every other value is refused, like the CUDA library.
// tests/test_ctu_driver_10bit.py checks it against the 10-bit reference (oracle/_ref/kvazaar_10b); ctu_hostsim.cpp stays
// the 8-bit host build of tests/test_ctu_driver.py.  Only tests/ may load the resulting library
// (tests/hostsim/libkvzctu_hostsim_10b.so); libkvzcuda.so never does.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <vector>
#include <mutex>
#include <condition_variable>

#include "../../include/kvz_cuda_ctu.h"
#include "../../kvazaar_b200/csrc/ctu/ctu_frame.h"

using namespace kvzctu;

static_assert(sizeof(kvz_cuda_ctu_config) == sizeof(CtuConfig), "config layout");
static_assert(sizeof(kvz_cuda_ctu_cu) == sizeof(CuRec), "cu layout");
static_assert(sizeof(kvz_cuda_ctu_sao) == sizeof(SaoRec), "sao layout");

struct Slot {
  bool busy = false;
  std::vector<uint8_t> src[3], rec[3], out[3], hor[3], ver[3], dbg[3];     // bytes: samples of the configured type
  std::vector<CuRec> cu;
  std::vector<int16_t> coeff;
  std::vector<SaoRec> sao;
  std::vector<CabacState> row_ctx;
  std::vector<uint8_t> dbg_ctx;
};

struct kvz_cuda_ctu_enc {
  CtuConfig cfg;
  int pix;                       // bytes per sample
  int wl, hl;
  CtuTables *T;
  void *W;                       // CtuWorkT<Pix>
  void *S;                       // CtuST<Pix>
  SaoStats *st;
  std::vector<Slot> slots;
  std::mutex mtx;                // one scratch set: pictures are searched one at a time
  std::condition_variable cv;
};

template <typename Pix> static FrameDevT<Pix> frame_of(kvz_cuda_ctu_enc *e, Slot &s)
{
  FrameDevT<Pix> F;
  F.src_y = (const Pix *)s.src[0].data(); F.src_u = (const Pix *)s.src[1].data(); F.src_v = (const Pix *)s.src[2].data();
  F.rec_y = (Pix *)s.rec[0].data(); F.rec_u = (Pix *)s.rec[1].data(); F.rec_v = (Pix *)s.rec[2].data();
  F.out_y = (Pix *)s.out[0].data(); F.out_u = (Pix *)s.out[1].data(); F.out_v = (Pix *)s.out[2].data();
  F.dbg_y = (Pix *)s.dbg[0].data(); F.dbg_u = (Pix *)s.dbg[1].data(); F.dbg_v = (Pix *)s.dbg[2].data();
  F.hor_y = (Pix *)s.hor[0].data(); F.hor_u = (Pix *)s.hor[1].data(); F.hor_v = (Pix *)s.hor[2].data();
  F.ver_y = (Pix *)s.ver[0].data(); F.ver_u = (Pix *)s.ver[1].data(); F.ver_v = (Pix *)s.ver[2].data();
  F.cu = s.cu.data(); F.coeff = s.coeff.data(); F.sao = s.sao.data(); F.row_ctx = s.row_ctx.data();
  F.cu_stride = e->wl * 16; F.wlcu = e->wl; F.hlcu = e->hl;
  return F;
}

// every CTU in coding order, then SAO over the picture
template <typename Pix> static void search_picture(kvz_cuda_ctu_enc *e, Slot &s)
{
  FrameDevT<Pix> F = frame_of<Pix>(e, s);
  CtxT<Pix> c = { e->T, &e->cfg, (CtuWorkT<Pix> *)e->W, (CtuST<Pix> *)e->S };
  for (int cy = 0; cy < F.hlcu; ++cy)
    for (int cx = 0; cx < F.wlcu; ++cx) {
      memcpy(&s.dbg_ctx[(size_t)(cy * F.wlcu + cx) * CTX_COUNT], s.row_ctx[cy].ctx, CTX_COUNT);
      ctu_job(c, &F, e->st, cx, cy);
    }
  for (int cy = 0; cy < F.hlcu; ++cy)
    for (int cx = 0; cx < F.wlcu; ++cx) ctu_sao_apply(&e->cfg, &F, cx, cy);
}

extern "C" {

int kvz_cuda_ctu_config_supported(const kvz_cuda_ctu_config *c)
{
  if (!c) return -1;
  if (c->width < 8 || c->height < 8 || (c->width & 7) || (c->height & 7)) return -1;
  if (c->rdo < 0 || c->rdo > 3) return -1;
  if (c->pu_depth_intra_min < 1 || c->pu_depth_intra_max > 4 || c->pu_depth_intra_min > c->pu_depth_intra_max) return -1;
  if (c->qp < 0 || c->qp > 51) return -1;
  if (c->bitdepth != 0 && c->bitdepth != 8 && c->bitdepth != 10) return -1;
  return 0;
}

kvz_cuda_ctu_enc *kvz_cuda_ctu_open(const kvz_cuda_ctu_config *cfg, int slots)
{
  if (kvz_cuda_ctu_config_supported(cfg)) return NULL;
  kvz_cuda_ctu_enc *e = new kvz_cuda_ctu_enc;
  memcpy(&e->cfg, cfg, sizeof(CtuConfig));
  e->pix = cfg->bitdepth == 10 ? 2 : 1;
  e->T = new CtuTables;
  ctu_tables_init(e->T);
  e->W = calloc(1, e->pix == 2 ? sizeof(CtuWorkT<uint16_t>) : sizeof(CtuWorkT<uint8_t>));
  e->S = calloc(1, e->pix == 2 ? sizeof(CtuST<uint16_t>) : sizeof(CtuST<uint8_t>));
  e->st = (SaoStats *)calloc(1, sizeof(SaoStats));
  e->slots.resize(slots > 0 ? slots : 1);
  const int W = cfg->width, H = cfg->height;
  e->wl = (W + 63) / 64; e->hl = (H + 63) / 64;
  const size_t px = (size_t)e->pix;
  for (Slot &s : e->slots) {
    for (int p = 0; p < 3; ++p) {
      const size_t pw = p ? W / 2 : W, ph = p ? H / 2 : H;
      s.src[p].assign(pw * ph * px, 0); s.rec[p].assign(pw * ph * px, 0); s.out[p].assign(pw * ph * px, 0); s.dbg[p].assign(pw * ph * px, 0);
      s.hor[p].assign(pw * e->hl * px, 0); s.ver[p].assign(ph * e->wl * px, 0);
    }
    s.cu.assign((size_t)(e->wl * 16) * (e->hl * 16), CuRec());
    s.coeff.assign((size_t)e->wl * e->hl * 6144, 0);
    s.sao.assign((size_t)e->wl * e->hl * 2, SaoRec());
    s.row_ctx.assign(e->hl, CabacState());
    s.dbg_ctx.assign((size_t)e->wl * e->hl * CTX_COUNT, 0);
  }
  return e;
}

void kvz_cuda_ctu_close(kvz_cuda_ctu_enc *e)
{
  if (!e) return;
  delete e->T; free(e->W); free(e->S); free(e->st);
  delete e;
}

int kvz_cuda_ctu_submit(kvz_cuda_ctu_enc *e, const uint8_t *y, const uint8_t *u, const uint8_t *v, int stride_y, int stride_c,
                        const uint8_t *ctx_init, double lambda, double lambda_sqrt, int qp)
{
  // like the CUDA library: blocks while every slot is busy
  std::unique_lock<std::mutex> lock(e->mtx);
  int id = -1;
  e->cv.wait(lock, [&] { for (size_t i = 0; i < e->slots.size(); ++i) if (!e->slots[i].busy) { id = (int)i; return true; } return false; });
  Slot &s = e->slots[id];
  s.busy = true;
  e->cfg.lambda = lambda; e->cfg.lambda_sqrt = lambda_sqrt; e->cfg.qp = qp;
  if (getenv("KVZ_CTU_DEBUG")) fprintf(stderr, "hostsim: qp %d lambda %.17g sqrt %.17g rdo %d pu %d-%d rdoq %d/%d sh %d ts %d sao %d dbk %d bitdepth %d\n", qp, lambda, lambda_sqrt, e->cfg.rdo, e->cfg.pu_depth_intra_min, e->cfg.pu_depth_intra_max, e->cfg.rdoq_enable, e->cfg.rdoq_skip, e->cfg.signhide_enable, e->cfg.trskip_enable, e->cfg.sao_type, e->cfg.deblock_enable, e->cfg.bitdepth);
  const size_t px = (size_t)e->pix, wb = (size_t)e->cfg.width * px, sy = (size_t)stride_y * px, sc = (size_t)stride_c * px;
  const int H = e->cfg.height;
  const uint8_t *yb = (const uint8_t *)y, *ub = (const uint8_t *)u, *vb = (const uint8_t *)v;
  for (int r = 0; r < H; ++r) memcpy(&s.src[0][(size_t)r * wb], yb + (size_t)r * sy, wb);
  for (int r = 0; r < H / 2; ++r) { memcpy(&s.src[1][(size_t)r * (wb / 2)], ub + (size_t)r * sc, wb / 2); memcpy(&s.src[2][(size_t)r * (wb / 2)], vb + (size_t)r * sc, wb / 2); }
  memset(s.cu.data(), 0, s.cu.size() * sizeof(CuRec));
  for (CabacState &c : s.row_ctx) { memcpy(c.ctx, ctx_init, CTX_COUNT); c.update = 0; }
  if (e->pix == 2) search_picture<uint16_t>(e, s);
  else search_picture<uint8_t>(e, s);
  return id;
}

int kvz_cuda_ctu_wait(kvz_cuda_ctu_enc *e, int slot, kvz_cuda_ctu_result *out)
{
  if (slot < 0 || slot >= (int)e->slots.size() || !e->slots[slot].busy) return -1;
  Slot &s = e->slots[slot];
  out->cu = (const kvz_cuda_ctu_cu *)s.cu.data();
  out->cu_stride = e->wl * 16;
  out->width_in_lcu = e->wl; out->height_in_lcu = e->hl;
  out->coeff = s.coeff.data();
  out->sao = (const kvz_cuda_ctu_sao *)s.sao.data();
  out->rec_y = s.out[0].data(); out->rec_u = s.out[1].data(); out->rec_v = s.out[2].data();
  out->dbg_ctx = s.dbg_ctx.data();
  out->dbg_y = s.dbg[0].data(); out->dbg_u = s.dbg[1].data(); out->dbg_v = s.dbg[2].data();
  return 0;
}

// "device" memory of the host build is host memory
int kvz_cuda_ctu_submit_device(kvz_cuda_ctu_enc *e, const uint8_t *y, const uint8_t *u, const uint8_t *v, int stride_y, int stride_c,
                               const uint8_t *ctx_init, double lambda, double lambda_sqrt, int qp)
{
  return kvz_cuda_ctu_submit(e, y, u, v, stride_y, stride_c, ctx_init, lambda, lambda_sqrt, qp);
}
int kvz_cuda_ctu_wait_device(kvz_cuda_ctu_enc *e, int slot, kvz_cuda_ctu_device_result *out)
{
  if (slot < 0 || slot >= (int)e->slots.size() || !e->slots[slot].busy) return -1;
  Slot &s = e->slots[slot];
  memset(out, 0, sizeof(*out));
  out->cu = (const kvz_cuda_ctu_cu *)s.cu.data(); out->coeff = s.coeff.data(); out->sao = (const kvz_cuda_ctu_sao *)s.sao.data();
  out->rec = s.out[0].data();
  out->cu_stride = e->wl * 16; out->width_in_lcu = e->wl; out->height_in_lcu = e->hl;
  return 0;
}

void kvz_cuda_ctu_release(kvz_cuda_ctu_enc *e, int slot)
{
  {
    std::lock_guard<std::mutex> lock(e->mtx);
    if (slot >= 0 && slot < (int)e->slots.size()) e->slots[slot].busy = false;
  }
  e->cv.notify_all();
}

uint64_t kvz_cuda_ctu_launches(const kvz_cuda_ctu_enc *) { return 0; }

}  // extern "C"
