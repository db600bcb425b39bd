// K16: the contrastive head (model/modeling.py:491-526) on the K1 tensor-core GEMM at fp32-grade accuracy.
// The features are fp32; every product x.y is taken as xh.yh + xh.yl + xl.yh with x = xh + xl (xh = bf16(x),
// xl = bf16(x - xh)), and the three terms are ONE K1 GEMM over a K concatenated three times:
//   logits   S[n, nW]     = [xh | xh | xl] . [yh | yl | yh]^T / temp             (K = 3 Cs)
//   d_x      [n, Cs]      = [dSh | dSh | dSl] . [yh ; yl ; yh]                    (K = 3 nW)
//   d_y_all  [nW, Cs]     = [dSh ; dSh ; dSl]^T . [xh ; xl ; xh]                  (K = 3 n)
// ("|" = side by side along a row, ";" = stacked rows).  These two kernels write those operands: the split of fp32 rows
// into three bf16 segments, and the row kernel that turns the logits into dS = coeff (softmax - onehot) / temp, written
// directly as its hi/lo operands in both layouts (dS never exists in fp32).  The GEMMs run without split-K, so the head
// is deterministic.
#include "host_common.h"
#include "ptx.cuh"

namespace mb {

__device__ __forceinline__ void split_bf16(float v, bf16& h, bf16& l) {
  h = __float2bfloat16_rn(v);
  l = __float2bfloat16_rn(v - __bfloat162float(h));
}

// out[s * seg_stride + r * ld + c] <- (lo_mask bit s ? lo : hi)(x[r * ldx + c]), s = 0, 1, 2
__global__ void ctr_split_kernel(const float* __restrict__ x, int rows, int C, int ldx, bf16* __restrict__ out, long long ld,
                                 long long seg_stride, int lo_mask) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)rows * C) return;
  const int r = (int)(i / C), c = (int)(i % C);
  bf16 h, l;
  split_bf16(x[(size_t)r * ldx + c], h, l);
  bf16* o = out + (size_t)r * ld + c;
#pragma unroll
  for (int s = 0; s < 3; ++s) o[s * seg_stride] = (lo_mask >> s) & 1 ? l : h;
}

// One block per row i of the logits: g = scale * coeff[i] * (exp(S[i, c] - lse[i]) - [c == label[i]]), g = gh + gl;
// row i of dsh <- [gh | gh | gl] (segment stride C), rows i, n + i, 2n + i of dsv <- gh, gh, gl.
__global__ void __launch_bounds__(256) ctr_dlogits_kernel(const float* __restrict__ logits, int ld, const int* __restrict__ labels,
                                                          int n, int C, const float* __restrict__ lse,
                                                          const float* __restrict__ coeff, float scale, bf16* __restrict__ dsh,
                                                          int ld_h, bf16* __restrict__ dsv, int ld_v) {
  const int r = blockIdx.x;
  const float* row = logits + (size_t)r * ld;
  const float l = lse[r], cf = coeff[r] * scale;
  const int lab = labels[r];
  bf16* h_row = dsh + (size_t)r * ld_h;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const float g = cf * (__expf(row[c] - l) - (c == lab ? 1.f : 0.f));
    bf16 gh, gl;
    split_bf16(g, gh, gl);
    h_row[c] = gh;
    h_row[C + c] = gh;
    h_row[2 * C + c] = gl;
    dsv[(size_t)r * ld_v + c] = gh;
    dsv[(size_t)(n + r) * ld_v + c] = gh;
    dsv[(size_t)(2 * n + r) * ld_v + c] = gl;
  }
}

}  // namespace mb

using namespace mb;

extern "C" int merlot_ctr_split(const float* x, int rows, int C, int ldx, void* out, long long ld, long long seg_stride, int lo_mask,
                                void* stream_) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
  MB_REQUIRE(x && out, MERLOT_EINVAL, "ctr_split: null pointer");
  MB_REQUIRE(rows >= 0 && C > 0 && ldx >= C && ld >= C && lo_mask >= 0 && lo_mask < 8, MERLOT_ESHAPE,
             "ctr_split: need C > 0, ldx >= C, ld >= C, 0 <= lo_mask < 8");
  if (rows == 0) return MERLOT_OK;
  const long long n = (long long)rows * C;
  ctr_split_kernel<<<(unsigned)ceil_div_ll(n, 256), 256, 0, st>>>(x, rows, C, ldx, reinterpret_cast<bf16*>(out), ld, seg_stride,
                                                                  lo_mask);
  MB_CHECK_LAUNCH();
  return MERLOT_OK;
}

extern "C" int merlot_ctr_dlogits(const float* logits, int ld, const int* labels, int rows, int C, const float* lse,
                                  const float* coeff, float scale, void* dsh, int ld_h, void* dsv, int ld_v, void* stream_) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
  MB_REQUIRE(logits && labels && lse && coeff && dsh && dsv, MERLOT_EINVAL, "ctr_dlogits: null pointer");
  MB_REQUIRE(C > 0 && ld >= C && ld_h >= 3 * C && ld_v >= C, MERLOT_ESHAPE, "ctr_dlogits: need 0 < C <= ld, ld_v and 3C <= ld_h");
  if (rows == 0) return MERLOT_OK;
  ctr_dlogits_kernel<<<rows, 256, 0, st>>>(logits, ld, labels, rows, C, lse, coeff, scale, reinterpret_cast<bf16*>(dsh), ld_h,
                                           reinterpret_cast<bf16*>(dsv), ld_v);
  MB_CHECK_LAUNCH();
  return MERLOT_OK;
}
