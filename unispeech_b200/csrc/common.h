// Host-side helpers shared by the C-ABI translation units: error reporting and launch checks.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

namespace b200 {

// thread-local last error string, exposed through b200s_last_error()
char* last_error_buf();
void set_last_error(const char* fmt, ...);

#define B200_CHECK_ARG(cond, ...)        \
  do {                                   \
    if (!(cond)) {                       \
      b200::set_last_error(__VA_ARGS__); \
      return -1;                         \
    }                                    \
  } while (0)

#define B200_CHECK_CUDA(expr)                                                                  \
  do {                                                                                         \
    cudaError_t _e = (expr);                                                                   \
    if (_e != cudaSuccess) {                                                                   \
      b200::set_last_error("%s:%d CUDA error %s: %s", __FILE__, __LINE__, cudaGetErrorName(_e), \
                           cudaGetErrorString(_e));                                            \
      return -2;                                                                               \
    }                                                                                          \
  } while (0)

// number of kernels this library has launched (read through b200s_launch_count(); bench.py reports it)
extern long long g_launch_count;
#define B200_CHECK_LAUNCH()              \
  do {                                   \
    ++b200::g_launch_count;              \
    B200_CHECK_CUDA(cudaGetLastError()); \
  } while (0)

// Launch with programmatic dependent launch enabled: the kernel's CTAs can be scheduled while the previous kernel of the
// stream is still draining; every kernel calls pdl_wait() (ptx.cuh) before its first global access.
template <typename... KArgs, typename... Args>
static inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                                     Args&&... args) {
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

static inline int ceil_div(int a, int b) { return (a + b - 1) / b; }
static inline long long ceil_div_ll(long long a, long long b) { return (a + b - 1) / b; }

// sm count of the current device (cached)
int sm_count();

}  // namespace b200
