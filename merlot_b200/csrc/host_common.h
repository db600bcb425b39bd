// Host-side helpers shared by all translation units of libmerlot_b200.so:
// error reporting (C-ABI returns int codes + thread-local message), launch counting, TMA tensor-map encoding.
#pragma once
#include <stdlib.h>
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../../include/merlot_b200.h"

namespace mb {

// thread-local message returned by merlot_last_error()
char* last_error_buf();
int set_error(int code, const char* fmt, ...);
void count_launch(int n = 1);

#define MB_CHECK_CUDA(expr)                                                                        \
  do {                                                                                             \
    cudaError_t _e = (expr);                                                                       \
    if (_e != cudaSuccess)                                                                         \
      return mb::set_error(MERLOT_ECUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), \
                           __FILE__, __LINE__);                                                   \
  } while (0)

#define MB_CHECK_LAUNCH()                                                                                      \
  do {                                                                                                         \
    cudaError_t _e = cudaGetLastError();                                                                       \
    if (_e != cudaSuccess)                                                                                     \
      return mb::set_error(MERLOT_ECUDA, "kernel launch failed: %s (%s:%d)", cudaGetErrorString(_e), __FILE__, \
                           __LINE__);                                                                          \
    mb::count_launch();                                                                                        \
  } while (0)

#define MB_REQUIRE(cond, code, ...)                      \
  do {                                                   \
    if (!(cond)) return mb::set_error(code, __VA_ARGS__); \
  } while (0)

// 2-D bf16 tensor map, 128B swizzle, zero OOB fill. dims/box are {inner, outer}; ld = outer stride in elements.
int make_tmap_bf16_2d(CUtensorMap* out, const void* base, uint64_t inner, uint64_t outer, uint64_t ld_elems,
                      uint32_t box_inner, uint32_t box_outer);
// 3-D bf16 tensor map (inner, mid, outer) with element strides ld_mid / ld_outer.
int make_tmap_bf16_3d(CUtensorMap* out, const void* base, uint64_t d0, uint64_t d1, uint64_t d2, uint64_t ld1,
                      uint64_t ld2, uint32_t b0, uint32_t b1, uint32_t b2);

int device_sms();  // SMs of the device
int num_sms();     // SMs the persistent kernels may fill (device_sms() minus merlot_set_sm_reserve)

// Launch with the programmatic-stream-serialization attribute (PDL). Kernels launched this way MUST call pdl_wait()
// before their first global-memory access.
template <typename... KArgs, typename... Args>
static inline cudaError_t launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  static const bool no_pdl = [] { const char* e = getenv("MERLOT_NO_PDL"); return e && e[0] == '1'; }();  // diagnostics: true per-kernel times
  cfg.attrs = at; cfg.numAttrs = no_pdl ? 0 : 1;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

static inline int ceil_div(int a, int b) { return (a + b - 1) / b; }
static inline long long ceil_div_ll(long long a, long long b) { return (a + b - 1) / b; }

}  // namespace mb
