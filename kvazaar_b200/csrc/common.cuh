// common.cuh -- shared device helpers and host-side plumbing for libkvzcuda (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <atomic>

#include "../../include/kvz_cuda.h"
#include "pixel_rules.h"

namespace kvzc {

using namespace kvzpix;       // sample traits and the sample-domain rules shared with the CTU search

// ---------------------------------------------------------------- host side
extern std::atomic<uint64_t> g_launches;
extern int g_device;        // -1 until kvz_cuda_init succeeds
extern int g_sm_count;
void set_error(const char *fmt, ...);

#define KVZC_CHECK(expr)                                                                   \
  do {                                                                                     \
    cudaError_t e__ = (expr);                                                              \
    if (e__ != cudaSuccess) {                                                              \
      kvzc::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__), __FILE__, __LINE__); \
      return KVZ_CUDA_E_RUNTIME;                                                           \
    }                                                                                      \
  } while (0)

#define KVZC_REQUIRE_DEVICE()                                                              \
  do {                                                                                     \
    if (kvzc::g_device < 0 && kvz_cuda_init(-1) != 0) return KVZ_CUDA_E_NODEVICE;          \
  } while (0)

#define KVZC_ARG(cond)                                                                     \
  do {                                                                                     \
    if (!(cond)) { kvzc::set_error("bad argument: %s (%s:%d)", #cond, __FILE__, __LINE__); return KVZ_CUDA_E_ARG; } \
  } while (0)

// count a launch and check it
#define KVZC_LAUNCHED()                                                                    \
  do {                                                                                     \
    kvzc::g_launches.fetch_add(1, std::memory_order_relaxed);                              \
    KVZC_CHECK(cudaGetLastError());                                                        \
  } while (0)

static inline cudaStream_t as_stream(void *s) { return (cudaStream_t)s; }

// Per-thread staging for the synchronous per-call strategy functions: one pinned host
// buffer + one device buffer + one stream per calling thread (the host calls strategies
// concurrently from every threadqueue worker, ref: threadqueue.c:275).
struct Staging {
  cudaStream_t stream = nullptr;
  uint8_t *h = nullptr;   // pinned
  uint8_t *d = nullptr;
  size_t cap = 0;
  int ensure(size_t bytes);
};
Staging &tls_staging();

// Lays out inputs/outputs of one call inside the staging buffers.
struct Call {
  Staging &s;
  size_t off = 0, in_end = 0;
  bool ok = true;
  explicit Call(size_t bytes) : s(tls_staging()) { ok = s.ensure(bytes + 4096) == 0; }
  size_t take(size_t bytes) { size_t o = off; off = (off + bytes + 255) & ~size_t(255); return o; }
  // contiguous input
  template <class T> T *in(const T *host, size_t n) {
    size_t o = take(n * sizeof(T));
    memcpy(s.h + o, host, n * sizeof(T));
    in_end = off;
    return (T *)(s.d + o);
  }
  // strided window (rows of `w` elements, host stride `stride`) -> compact stride w
  template <class T> T *in2d(const T *host, int w, int h, long stride) {
    size_t o = take((size_t)w * h * sizeof(T));
    T *dst = (T *)(s.h + o);
    for (int y = 0; y < h; ++y) memcpy(dst + (size_t)y * w, host + (long)y * stride, (size_t)w * sizeof(T));
    in_end = off;
    return (T *)(s.d + o);
  }
  template <class T> T *host_ptr(T *dev) { return (T *)(s.h + ((uint8_t *)dev - s.d)); }
  size_t out_begin = 0;
  template <class T> T *out(size_t n) {
    if (!out_begin) out_begin = off;
    size_t o = take(n * sizeof(T));
    return (T *)(s.d + o);
  }
  int upload() {
    if (in_end) KVZC_CHECK(cudaMemcpyAsync(s.d, s.h, in_end, cudaMemcpyHostToDevice, s.stream));
    return 0;
  }
  int download() {
    if (off > out_begin)
      KVZC_CHECK(cudaMemcpyAsync(s.h + out_begin, s.d + out_begin, off - out_begin, cudaMemcpyDeviceToHost, s.stream));
    KVZC_CHECK(cudaStreamSynchronize(s.stream));
    return 0;
  }
};

// rdoq.cu: kvz_rdoq in place on the coefficients of the TUs of width n (used by the quantize_residual RDOQ branch)
int rdoq_launch_tus(const kvz_cuda_rdoq_params &p, const kvz_cuda_cabac_ctx *ctx_dev, int16_t *coeff, const kvz_cuda_tu *tus, int count, int n,
                    cudaStream_t st);

int rdoq_launch_grid(const kvz_cuda_rdoq_params &p, const kvz_cuda_cabac_ctx *ctx_dev, int16_t *coeff, int16_t *coeff2, int count, int log2n,
                     const int8_t *modes, int is_chroma, int tr_depth, cudaStream_t st);   // coeff2: second plane (V) or NULL

// coeff_cost.cu: CABAC bit cost of every TU of a uniform grid (frame-level pass)
int coeff_cost_launch_grid(int signhide, const kvz_cuda_cabac_ctx *ctx_dev, const int16_t *coeff, const int16_t *coeff2, int count, int log2n,
                           const int8_t *modes, int trskip_enable, double *bits_out, double *bits_out2, cudaStream_t st, int is_chroma = 0);

// ---------------------------------------------------------------- device side
__device__ __forceinline__ int warp_sum(int v)
{
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// block-wide integer sum; result valid in thread 0.  blockDim.x multiple of 32, <= 1024.
__device__ __forceinline__ int block_sum(int v)
{
  __shared__ int red[32];
  v = warp_sum(v);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  __syncthreads();
  if (lane == 0) red[wid] = v;
  __syncthreads();
  const int nw = (blockDim.x + 31) >> 5;
  v = (threadIdx.x < nw) ? red[threadIdx.x] : 0;
  if (wid == 0) v = warp_sum(v);
  return v;
}

__device__ __forceinline__ int clip3(int lo, int hi, int v) { return min(max(v, lo), hi); }

// the five offsets of an SAO edge class (categories 0..4) in registers, looked up by selection: an array indexed at run
// time would live in local memory
struct EdgeOffsets {
  int o[5];
  __device__ __forceinline__ int operator[](int cat) const
  {
    int v = o[0];
#pragma unroll
    for (int k = 1; k < 5; ++k) v = cat == k ? o[k] : v;
    return v;
  }
};

}  // namespace kvzc
