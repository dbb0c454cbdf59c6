// Definitions of the shared host helpers (host.cuh) and of the library-wide C ABI entry points.
#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <string>

#include "host.cuh"

static thread_local std::string g_err;

extern "C" int mvb_abi_version(void) { return MVB_ABI_VERSION; }
extern "C" const char* mvb_last_error(void) { return g_err.c_str(); }

namespace mvb {

int set_error(int code, const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  g_err = buf;
  return code;
}

int check_offsets(const uint64_t* off, size_t n, size_t arena_bytes, const char* what) {
  for (size_t i = 0; i < n; ++i)
    if (off[i] % 16 || off[i] >= arena_bytes)
      return set_error(MVB_ERR_ARG, "%s %llu not 16B-aligned or outside the arena", what, (unsigned long long)off[i]);
  return MVB_OK;
}

// SM cap of mvb_test_set_sm_limit (0: none).  It only ever lowers the count: the persistent kernel and the split-K
// GEMM need every CTA of their grid co-resident, which a count above the device's own would break.
static std::atomic<int> g_sm_limit{0};

int current_device(int* dev, int* n_sm) {
  MVB_CK(cudaGetDevice(dev));
  MVB_CK(cudaDeviceGetAttribute(n_sm, cudaDevAttrMultiProcessorCount, *dev));
  const int cap = g_sm_limit.load();
  if (cap > 0 && cap < *n_sm) *n_sm = cap;
  return MVB_OK;
}

}  // namespace mvb

extern "C" int mvb_test_set_sm_limit(int32_t n) {
  if (n < 0) return mvb::set_error(MVB_ERR_ARG, "mvb_test_set_sm_limit: n = %d must be >= 0", n);
  mvb::g_sm_limit.store(n);
  return MVB_OK;
}
