// Status strings, version and per-thread CUDA error text for the dgcn C ABI.
#include <stdio.h>
#include <atomic>
#include <mutex>
#include <string>
#include <vector>
#include "common.cuh"

namespace dgcn {
static thread_local char g_last_error[512] = "";
void set_last_cuda_error(cudaError_t e, const char* file, int line) {
  snprintf(g_last_error, sizeof(g_last_error), "%s (%s) at %s:%d", cudaGetErrorName(e), cudaGetErrorString(e), file,
           line);
  (void)cudaGetLastError();   // reported through the status code: do not leave it for an unrelated later launch check
}

static int device_attr(cudaDeviceAttr attr, std::atomic<int>* cache, int fallback) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return fallback;
  int v = cache[dev].load(std::memory_order_relaxed);
  if (v > 0) return v;
  if (cudaDeviceGetAttribute(&v, attr, dev) != cudaSuccess || v <= 0) return fallback;
  cache[dev].store(v, std::memory_order_relaxed);
  return v;
}
int device_sm_count() {
  static std::atomic<int> cache[64];
  return device_attr(cudaDevAttrMultiProcessorCount, cache, 132);
}
size_t device_l2_bytes() {
  static std::atomic<int> cache[64];
  return static_cast<size_t>(device_attr(cudaDevAttrL2CacheSize, cache, 50 << 20));
}

static std::atomic<int> g_cert_on{0};
static std::atomic<int64_t> g_cert_failed{0}, g_cert_queries{0};
bool debug_certification_on() { return g_cert_on.load(std::memory_order_relaxed) != 0; }
void debug_certification_add(int64_t uncertified, int64_t queries) {
  g_cert_failed.fetch_add(uncertified, std::memory_order_relaxed);
  g_cert_queries.fetch_add(queries, std::memory_order_relaxed);
}

struct TimedLaunch {
  std::string tag;
  cudaEvent_t beg, end;
};
static std::mutex g_timing_mu;
static std::atomic<int> g_timing_on{0};
static std::vector<TimedLaunch*> g_timed;

KernelTimer::KernelTimer(cudaStream_t stream, const char* tag) : stream_(stream), slot_(nullptr) {
  if (!g_timing_on.load(std::memory_order_relaxed)) return;
  TimedLaunch* t = new TimedLaunch();
  t->tag = tag;
  if (cudaEventCreate(&t->beg) != cudaSuccess || cudaEventCreate(&t->end) != cudaSuccess) {
    delete t;
    return;
  }
  cudaEventRecord(t->beg, stream);
  slot_ = t;
}
KernelTimer::~KernelTimer() {
  if (!slot_) return;
  TimedLaunch* t = static_cast<TimedLaunch*>(slot_);
  cudaEventRecord(t->end, stream_);
  std::lock_guard<std::mutex> lk(g_timing_mu);
  g_timed.push_back(t);
}
}  // namespace dgcn

extern "C" {
int dgcn_debug_kernel_timing(int32_t enable) {
  return dgcn::g_timing_on.exchange(enable ? 1 : 0);
}
int dgcn_debug_kernel_timing_read(const char* tag, double* total_ms, int64_t* launches) {
  if (!tag || !total_ms || !launches) return DGCN_ERR_BAD_ARG;
  std::lock_guard<std::mutex> lk(dgcn::g_timing_mu);
  double ms = 0.0;
  int64_t n = 0;
  std::vector<dgcn::TimedLaunch*> keep;
  for (dgcn::TimedLaunch* t : dgcn::g_timed) {
    if (t->tag != tag) {
      keep.push_back(t);
      continue;
    }
    float one = 0.f;
    if (cudaEventSynchronize(t->end) == cudaSuccess && cudaEventElapsedTime(&one, t->beg, t->end) == cudaSuccess) {
      ms += one;
      ++n;
    }
    cudaEventDestroy(t->beg);
    cudaEventDestroy(t->end);
    delete t;
  }
  dgcn::g_timed.swap(keep);
  *total_ms = ms;
  *launches = n;
  return DGCN_OK;
}
int dgcn_debug_tc_certification(int32_t enable) {
  return dgcn::g_cert_on.exchange(enable ? 1 : 0);
}
int dgcn_debug_tc_certification_read(int64_t* uncertified, int64_t* queries) {
  if (!uncertified || !queries) return DGCN_ERR_BAD_ARG;
  *uncertified = dgcn::g_cert_failed.exchange(0);
  *queries = dgcn::g_cert_queries.exchange(0);
  return DGCN_OK;
}
int dgcn_version(void) { return 200; }
const char* dgcn_status_string(int status) {
  switch (status) {
    case DGCN_OK: return "ok";
    case DGCN_ERR_BAD_ARG: return "bad argument (null pointer or inconsistent size)";
    case DGCN_ERR_UNSUPPORTED: return "request outside what the sm_90a kernels cover";
    case DGCN_ERR_WORKSPACE: return "workspace too small";
    case DGCN_ERR_CUDA: return "CUDA launch failed";
    case DGCN_ERR_REDUCE: return "cross-rank reduction of the BatchNorm statistics failed (reduce callback)";
    default: return "unknown status";
  }
}
const char* dgcn_last_cuda_error(void) { return dgcn::g_last_error; }
}
