// core.cu -- lifecycle, error reporting, memory helpers, per-thread staging.
#include <stdarg.h>
#include <stdlib.h>

#include <mutex>

#include "common.cuh"

namespace kvzc {
std::atomic<uint64_t> g_launches{0};
int g_device = -1;
int g_sm_count = 0;
static std::mutex g_mu;
static thread_local char g_err[512] = "";

void set_error(const char *fmt, ...)
{
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int Staging::ensure(size_t bytes)
{
  if (kvzc::g_device < 0 && kvz_cuda_init(-1) != 0) return KVZ_CUDA_E_NODEVICE;
  if (!stream) {
    KVZC_CHECK(cudaSetDevice(g_device));
    KVZC_CHECK(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
  }
  if (bytes > cap) {
    size_t ncap = cap ? cap : (size_t)1 << 20;
    while (ncap < bytes) ncap <<= 1;
    if (h) cudaFreeHost(h);
    if (d) cudaFree(d);
    h = d = nullptr; cap = 0;
    KVZC_CHECK(cudaHostAlloc((void **)&h, ncap, cudaHostAllocDefault));
    KVZC_CHECK(cudaMalloc((void **)&d, ncap));
    cap = ncap;
  }
  return 0;
}

Staging &tls_staging()
{
  static thread_local Staging s;
  return s;
}
}  // namespace kvzc

using namespace kvzc;

extern "C" {

int kvz_cuda_init(int device)
{
  std::lock_guard<std::mutex> lk(g_mu);
  if (g_device >= 0) return 0;
  // The CTU driver keeps one stream per picture in flight, and a picture's work is a dependent chain (copy, search
  // launch, SAO launch, copies back): streams that share a hardware queue run one picture at a time.  The default of 8
  // queues caps the pictures that really overlap at 8; ask for the maximum before the context exists (no effect, and no
  // harm, when the host process created it already).
  setenv("CUDA_DEVICE_MAX_CONNECTIONS", "32", 0);
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n == 0) {
    set_error("no CUDA device: %s", e == cudaSuccess ? "device count is 0" : cudaGetErrorString(e));
    return KVZ_CUDA_E_NODEVICE;
  }
  if (device < 0) {
    const char *env = getenv("KVZ_CUDA_DEVICE");
    if (env) device = atoi(env);
    else if (cudaGetDevice(&device) != cudaSuccess) device = 0;
  }
  if (device >= n) { set_error("device %d out of range (%d devices)", device, n); return KVZ_CUDA_E_ARG; }
  KVZC_CHECK(cudaSetDevice(device));
  cudaDeviceProp prop;
  KVZC_CHECK(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0) {
    set_error("libkvzcuda is built for sm_90a (H100) only; device %d is sm_%d%d", device, prop.major, prop.minor);
    return KVZ_CUDA_E_NODEVICE;
  }
  g_sm_count = prop.multiProcessorCount;
  g_device = device;
  return 0;
}

void kvz_cuda_shutdown(void) { std::lock_guard<std::mutex> lk(g_mu); g_device = -1; }
int kvz_cuda_available(void) { return g_device >= 0 || kvz_cuda_init(-1) == 0; }
const char *kvz_cuda_last_error(void) { return g_err; }
int kvz_cuda_sm_count(void) { return g_sm_count; }
uint64_t kvz_cuda_launch_count(void) { return g_launches.load(); }
int kvz_cuda_sync(void *stream) { KVZC_CHECK(cudaStreamSynchronize(as_stream(stream))); return 0; }

void *kvz_cuda_malloc(size_t bytes)
{
  if (g_device < 0 && kvz_cuda_init(-1) != 0) return nullptr;
  void *p = nullptr;
  if (cudaMalloc(&p, bytes) != cudaSuccess) { set_error("cudaMalloc(%zu) failed", bytes); return nullptr; }
  return p;
}
void kvz_cuda_free(void *p) { if (p) cudaFree(p); }
void *kvz_cuda_host_alloc(size_t bytes)
{
  if (g_device < 0 && kvz_cuda_init(-1) != 0) return nullptr;
  void *p = nullptr;
  if (cudaHostAlloc(&p, bytes, cudaHostAllocDefault) != cudaSuccess) { set_error("cudaHostAlloc(%zu) failed", bytes); return nullptr; }
  return p;
}
void kvz_cuda_host_free(void *p) { if (p) cudaFreeHost(p); }
int kvz_cuda_memcpy_h2d(void *dst, const void *src, size_t bytes, void *stream)
{
  KVZC_CHECK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, as_stream(stream)));
  return 0;
}
int kvz_cuda_memcpy_d2h(void *dst, const void *src, size_t bytes, void *stream)
{
  KVZC_CHECK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, as_stream(stream)));
  return 0;
}

}  // extern "C"
