// core.cu — ABI version, thread-local error string, launch counter.
#include <stdarg.h>
#include <string.h>
#include "common.cuh"

namespace b2ctr {
static thread_local char g_err[512] = "";
std::atomic<long long> g_launches{0};
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

static unsigned long long* g_oob[64] = {nullptr};
unsigned long long* oob_counter() {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return nullptr;
  if (!g_oob[dev]) {
    // cudaMalloc is illegal while the calling thread captures a graph: the counter is created by the first
    // (eager) launch of a model, long before its step is captured
    unsigned long long* p = nullptr;
    if (cudaMalloc(&p, sizeof(unsigned long long)) != cudaSuccess) { cudaGetLastError(); return nullptr; }
    cudaMemset(p, 0, sizeof(unsigned long long));
    g_oob[dev] = p;
  }
  return g_oob[dev];
}
}  // namespace b2ctr

extern "C" {
int32_t b2ctr_abi_version(void) { return 2; }
b2ctr_status_t b2ctr_embed_oob_count(int64_t* count, int32_t reset, void* stream) {
  B2_REQUIRE(count, "embed_oob_count: NULL count");
  unsigned long long* d = b2ctr::oob_counter();
  *count = 0;
  if (!d) return B2CTR_OK;
  unsigned long long h = 0;
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e = cudaMemcpyAsync(&h, d, sizeof(h), cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess && reset && true) e = cudaMemsetAsync(d, 0, sizeof(h), st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) {
    b2ctr::set_error("embed_oob_count: %s", cudaGetErrorString(e));
    cudaGetLastError();
    return B2CTR_ERR_CUDA;
  }
  *count = (int64_t)h;
  return B2CTR_OK;
}
const char* b2ctr_last_error(void) { return b2ctr::g_err; }
int64_t b2ctr_launch_count(void) { return (int64_t)b2ctr::g_launches.load(); }
void b2ctr_reset_launch_count(void) { b2ctr::g_launches.store(0); }
b2ctr_status_t b2ctr_enable_peer_access(int32_t peer_device) {
  cudaError_t e = cudaDeviceEnablePeerAccess(peer_device, 0);
  if (e == cudaErrorPeerAccessAlreadyEnabled) {
    cudaGetLastError();
    return B2CTR_OK;
  }
  if (e != cudaSuccess) {
    b2ctr::set_error("enable_peer_access(%d): %s", peer_device, cudaGetErrorString(e));
    cudaGetLastError();
    return B2CTR_ERR_CUDA;
  }
  return B2CTR_OK;
}
}
