// Host-side policies shared by the translation units of the C ABI (include/mvb200.h): error reporting, workspace
// layout, handle construction and graph capture.  Device helpers live in common.cuh.
#pragma once
#include <cuda_runtime.h>

#include <memory>

#include "../../include/mvb200.h"

namespace mvb {

// Records a printf-style message for mvb_last_error() (per thread) and returns `code`.
int set_error(int code, const char* fmt, ...);

#define MVB_CK(expr)                                                                                                  \
  do {                                                                                                                \
    cudaError_t _e = (expr);                                                                                          \
    if (_e != cudaSuccess)                                                                                            \
      return mvb::set_error(MVB_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
  } while (0)

// Grid width of the grid-stride element-wise launches (MBD, audio post).  A launch width, not an SM count: those
// kernels loop until they have covered their range, so the value only affects speed.
constexpr int GRID_STRIDE_CTAS = 148;

// Bump allocator over a caller's workspace: slices in the order taken, each 256-byte aligned; `end` is the total size.
struct WsBump {
  size_t end = 0;
  size_t take(size_t bytes) { const size_t at = end; end = (end + bytes + 255) / 256 * 256; return at; }
};

// MVB_ERR_ARG unless every arena offset is 16-byte aligned (TMA, 128-bit loads) and inside the arena.
int check_offsets(const uint64_t* off, size_t n, size_t arena_bytes, const char* what);

// The current device and its SM count (MVB_ERR_CUDA if a query fails).
int current_device(int* dev, int* n_sm);

// A handle under construction in mvb_*_create: freed through the module's mvb_*_destroy, which accepts a half-built
// handle, on every early return until release() hands it to the caller.
template <class H>
using Building = std::unique_ptr<H, int (*)(H*)>;

// Captures body(cap) on the capture stream `cap` and instantiates it into *exec (written only on success).  Returns
// body's own error, or MVB_ERR_CUDA if capture or instantiation fails.
template <class Body>
int capture_graph(cudaStream_t cap, cudaGraphExec_t* exec, Body body) {
  MVB_CK(cudaStreamBeginCapture(cap, cudaStreamCaptureModeThreadLocal));
  const int rc = body(cap);
  cudaGraph_t g = nullptr;
  cudaError_t e = cudaStreamEndCapture(cap, &g);
  cudaGraphExec_t ge = nullptr;
  if (rc == MVB_OK && e == cudaSuccess) e = cudaGraphInstantiate(&ge, g, 0);
  if (g) cudaGraphDestroy(g);
  if (rc != MVB_OK) return rc;
  if (e != cudaSuccess) return set_error(MVB_ERR_CUDA, "CUDA graph capture failed: %s", cudaGetErrorString(e));
  *exec = ge;
  return MVB_OK;
}

}  // namespace mvb
