#include "host_common.h"

#include <stdarg.h>

#include <atomic>
#include <mutex>

namespace mb {

static thread_local char g_err[512] = "";
static std::atomic<long long> g_launches{0};

char* last_error_buf() { return g_err; }

int set_error(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

static std::atomic<int> g_sm_reserve{0};

// SMs the persistent kernels (K1, K3) may fill.  With data parallelism NCCL's collective CTAs each occupy a whole SM for
// milliseconds; a persistent kernel launched with one CTA per SM then has CTAs that cannot start until others have finished
// and, with a static tile schedule, takes up to twice as long.  merlot_set_sm_reserve(n) leaves n SMs to the collective.
// SMs of the current device (132 on an H100 SXM), independent of the reserve below: for workspace sizes and fixed grids.
int device_sms() {
  static int sms = 0;
  if (sms == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 132;
    if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0) sms = 132;
  }
  return sms;
}

int num_sms() {
  const int sms = device_sms();
  const int r = g_sm_reserve.load(std::memory_order_relaxed);
  return (r > 0 && r < sms - 8) ? sms - r : sms;
}

// cuTensorMapEncodeTiled is a driver-API symbol; resolve it through the runtime so the library has no link-time
// dependency on libcuda.so (the build container has no driver).
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode() {
  static PFN_encodeTiled fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_encodeTiled>(p);
  });
  return fn;
}

static int make_tmap_2d(CUtensorMap* out, CUtensorMapDataType dtype, uint64_t elem_bytes, const void* base, uint64_t inner,
                        uint64_t outer, uint64_t ld_elems, uint32_t box_inner, uint32_t box_outer) {
  PFN_encodeTiled enc = get_encode();
  if (!enc) return set_error(MERLOT_ECUDA, "cuTensorMapEncodeTiled entry point not available (no CUDA driver?)");
  cuuint64_t dims[2] = {inner, outer};
  cuuint64_t strides[1] = {ld_elems * elem_bytes};
  cuuint32_t box[2] = {box_inner, box_outer};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(out, dtype, 2, const_cast<void*>(base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return set_error(MERLOT_ECUDA,
                     "cuTensorMapEncodeTiled(2d) failed: CUresult %d (base=%p inner=%llu outer=%llu ld=%llu box=%ux%u)",
                     (int)r, base, (unsigned long long)inner, (unsigned long long)outer, (unsigned long long)ld_elems,
                     box_inner, box_outer);
  return MERLOT_OK;
}

int make_tmap_bf16_2d(CUtensorMap* out, const void* base, uint64_t inner, uint64_t outer, uint64_t ld_elems,
                      uint32_t box_inner, uint32_t box_outer) {
  return make_tmap_2d(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, base, inner, outer, ld_elems, box_inner, box_outer);
}

int make_tmap_f32_2d(CUtensorMap* out, const void* base, uint64_t inner, uint64_t outer, uint64_t ld_elems,
                     uint32_t box_inner, uint32_t box_outer) {
  return make_tmap_2d(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, base, inner, outer, ld_elems, box_inner, box_outer);
}

int make_tmap_bf16_3d(CUtensorMap* out, const void* base, uint64_t d0, uint64_t d1, uint64_t d2, uint64_t ld1,
                      uint64_t ld2, uint32_t b0, uint32_t b1, uint32_t b2) {
  PFN_encodeTiled enc = get_encode();
  if (!enc) return set_error(MERLOT_ECUDA, "cuTensorMapEncodeTiled entry point not available (no CUDA driver?)");
  cuuint64_t dims[3] = {d0, d1, d2};
  cuuint64_t strides[2] = {ld1 * 2, ld2 * 2};
  cuuint32_t box[3] = {b0, b1, b2};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return set_error(MERLOT_ECUDA, "cuTensorMapEncodeTiled(3d) failed: CUresult %d", (int)r);
  return MERLOT_OK;
}

}  // namespace mb

extern "C" void merlot_set_sm_reserve(int n) { mb::g_sm_reserve.store(n < 0 ? 0 : n); }
extern "C" const char* merlot_last_error(void) { return mb::last_error_buf(); }
extern "C" int merlot_abi_version(void) { return 1; }
extern "C" long long merlot_launch_count(void) { return mb::g_launches.load(); }
extern "C" void merlot_reset_launch_count(void) { mb::g_launches.store(0); }
