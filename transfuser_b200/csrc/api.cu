// Library-level entry points of the C-ABI: version, last-error text; the per-stream reduction scratch (common.cuh TfbScratch).
#include "common.cuh"
#include <string.h>

#include <mutex>
#include <unordered_map>
#include <vector>

namespace {
struct StreamScratch {
  float* f = nullptr;
  size_t nf = 0;
  unsigned int* cnt = nullptr;
  size_t nc = 0;
};
std::mutex g_scratch_mu;
std::unordered_map<cudaStream_t, StreamScratch> g_scratch;
std::vector<void*> g_retired;   // grown-out buffers: a captured CUDA graph may still use them

// cudaMalloc outside any stream capture in progress on this thread (the allocation is not a stream operation; graph capture in
// the global mode would reject it)
cudaError_t malloc_uncaptured(void** p, size_t bytes) {
  cudaStreamCaptureMode mode = cudaStreamCaptureModeRelaxed;
  cudaThreadExchangeStreamCaptureMode(&mode);
  const cudaError_t e = cudaMalloc(p, bytes);
  cudaThreadExchangeStreamCaptureMode(&mode);
  return e;
}
}  // namespace

int tfb_scratch(TfbScratch& w, size_t floats, size_t counters, cudaStream_t s) {
  std::lock_guard<std::mutex> lock(g_scratch_mu);
  StreamScratch& sc = g_scratch[s];
  if (floats > sc.nf) {
    const size_t n = floats > 2 * sc.nf ? floats : 2 * sc.nf;
    void* p = nullptr;
    if (malloc_uncaptured(&p, n * sizeof(float)) != cudaSuccess) { tfb_set_last_error("cudaMalloc(reduction scratch) failed"); return TFB_ERR_DRIVER; }
    if (sc.f) g_retired.push_back(sc.f);
    sc.f = static_cast<float*>(p);
    sc.nf = n;
  }
  if (counters > sc.nc) {
    const size_t n = counters > 4096 ? counters : 4096;
    void* p = nullptr;
    if (malloc_uncaptured(&p, n * sizeof(unsigned int)) != cudaSuccess) { tfb_set_last_error("cudaMalloc(reduction counters) failed"); return TFB_ERR_DRIVER; }
    if (cudaMemsetAsync(p, 0, n * sizeof(unsigned int), s) != cudaSuccess) { tfb_set_last_error("cudaMemsetAsync(reduction counters) failed"); return TFB_ERR_DRIVER; }
    if (sc.cnt) g_retired.push_back(sc.cnt);
    sc.cnt = static_cast<unsigned int*>(p);
    sc.nc = n;
  }
  w.f = sc.f;
  w.cnt = sc.cnt;
  return TFB_OK;
}

static thread_local char g_last_error[512] = "";

void tfb_set_last_error(const char* msg) {
  strncpy(g_last_error, msg ? msg : "", sizeof(g_last_error) - 1);
  g_last_error[sizeof(g_last_error) - 1] = 0;
}

TFB_API const char* tfb_last_error(void) { return g_last_error; }
TFB_API int tfb_abi_version(void) { return 1; }
