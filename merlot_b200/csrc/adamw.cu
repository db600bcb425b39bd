// K10: fused AdamW over the flat parameter arena (one launch per hyper-parameter group instead of one XLA computation
// per variable).  Restates utils/optimization.py:339-416 (AdamOptimizer.apply_gradients) including the bf16 first
// moment and the sign-bit-packed bf16 second moment (_decode_v/_encode_v, :267-288):
//   g2 = g*g + 1e-30;  m' = b1*m + (1-b1)*g;  v' = b2*v + (1-b2)*g2;  u = m'/(sqrt(v')+eps);  u += wd*p (wd>0);
//   p' = p - lr_t*u;   m' -> bf16 (RNE);  v' -> e=bf16(v'), stored as +e if |e-v'| <= |e*1.00390625-v'| else -e.
// g is first scaled by grad_scale (= 1/world_size: CrossShardOptimizer's mean, :241-245).
// Also emits the bf16 compute copy of the new parameter (bfloat16_getter, utils/model_utils.py:572-602) and can zero
// the gradient for the next step.  HBM traffic: 20 B/param (+2 bf16 copy, +4 grad zeroing).
// Explicit round-to-nearest intrinsics keep the op-by-op fp32 rounding of the reference (no FMA contraction), so the
// stored bf16 moments are bit-exact against the oracle.
#include "host_common.h"
#include "ptx.cuh"

namespace mb {

struct AdamDev {
  float* p; float* g; bf16* m; bf16* v; bf16* p_bf16;
  long long n;
  float b1, omb1, b2, omb2, eps, lr_t, wd, grad_scale;
  int zero_grad;
};

__device__ __forceinline__ void adam_elem(float& p, float g, bf16& mb, bf16& vb, const AdamDev& a) {
  g = __fmul_rn(g, a.grad_scale);
  const float g2 = __fadd_rn(__fmul_rn(g, g), 1e-30f);
  const float m = __bfloat162float(mb);
  const float vs = __bfloat162float(vb);
  const float vabs = fabsf(vs);
  const float v = vs > 0.f ? vabs : __fmul_rn(vabs, 1.00390625f);
  const float nm = __fadd_rn(__fmul_rn(a.b1, m), __fmul_rn(a.omb1, g));
  const float nv = __fadd_rn(__fmul_rn(a.b2, v), __fmul_rn(a.omb2, g2));
  float u = __fdiv_rn(nm, __fadd_rn(__fsqrt_rn(nv), a.eps));
  if (a.wd > 0.f) u = __fadd_rn(u, __fmul_rn(a.wd, p));
  p = __fsub_rn(p, __fmul_rn(a.lr_t, u));
  mb = __float2bfloat16_rn(nm);
  const bf16 e = __float2bfloat16_rn(nv);
  const float ef = __bfloat162float(e);
  const float err0 = fabsf(__fsub_rn(ef, nv));
  const float err1 = fabsf(__fsub_rn(__fmul_rn(ef, 1.00390625f), nv));
  vb = (err0 <= err1) ? e : __float2bfloat16_rn(-ef);
}

__global__ void __launch_bounds__(256) adamw_kernel(const AdamDev a) {
  const long long i8 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * 8;
  if (i8 >= a.n) return;
  if (i8 + 8 <= a.n) {
    float4 p0 = *reinterpret_cast<float4*>(a.p + i8), p1 = *reinterpret_cast<float4*>(a.p + i8 + 4);
    float4 g0 = *reinterpret_cast<float4*>(a.g + i8), g1 = *reinterpret_cast<float4*>(a.g + i8 + 4);
    uint4 mu = *reinterpret_cast<uint4*>(a.m + i8), vu = *reinterpret_cast<uint4*>(a.v + i8);
    float pv[8] = {p0.x, p0.y, p0.z, p0.w, p1.x, p1.y, p1.z, p1.w};
    const float gv[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
    bf16* mm = reinterpret_cast<bf16*>(&mu);
    bf16* vv = reinterpret_cast<bf16*>(&vu);
#pragma unroll
    for (int k = 0; k < 8; ++k) adam_elem(pv[k], gv[k], mm[k], vv[k], a);
    *reinterpret_cast<float4*>(a.p + i8) = make_float4(pv[0], pv[1], pv[2], pv[3]);
    *reinterpret_cast<float4*>(a.p + i8 + 4) = make_float4(pv[4], pv[5], pv[6], pv[7]);
    *reinterpret_cast<uint4*>(a.m + i8) = mu;
    *reinterpret_cast<uint4*>(a.v + i8) = vu;
    if (a.p_bf16)
      *reinterpret_cast<uint4*>(a.p_bf16 + i8) =
          make_uint4(pack_bf16x2(pv[0], pv[1]), pack_bf16x2(pv[2], pv[3]), pack_bf16x2(pv[4], pv[5]), pack_bf16x2(pv[6], pv[7]));
    if (a.zero_grad) {
      *reinterpret_cast<float4*>(a.g + i8) = make_float4(0.f, 0.f, 0.f, 0.f);
      *reinterpret_cast<float4*>(a.g + i8 + 4) = make_float4(0.f, 0.f, 0.f, 0.f);
    }
  } else {
    for (long long i = i8; i < a.n; ++i) {
      float pv = a.p[i];
      bf16 mm = a.m[i], vv = a.v[i];
      adam_elem(pv, a.g[i], mm, vv, a);
      a.p[i] = pv; a.m[i] = mm; a.v[i] = vv;
      if (a.p_bf16) a.p_bf16[i] = __float2bfloat16_rn(pv);
      if (a.zero_grad) a.g[i] = 0.f;
    }
  }
}

// tf.clip_by_global_norm (utils/optimization.py:233-237): norm = sqrt(sum g^2) over the whole arena, then
// g *= clip_norm / max(norm, clip_norm).  Two launches; the norm stays on the device (also reported as gradnorms/_overall).
__global__ void __launch_bounds__(256) sumsq_kernel(const float* __restrict__ g, long long n, double* __restrict__ acc) {
  __shared__ double sred[8];
  double s = 0.0;
  for (long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * 4; i < n; i += (long long)gridDim.x * blockDim.x * 4) {
    if (i + 4 <= n) {
      const float4 v = *reinterpret_cast<const float4*>(g + i);
      s += (double)v.x * v.x + (double)v.y * v.y + (double)v.z * v.z + (double)v.w * v.w;
    } else {
      for (long long j = i; j < n; ++j) s += (double)g[j] * g[j];
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) sred[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int w = 0; w < 8; ++w) t += sred[w];
    atomicAdd(acc, t);
  }
}
__global__ void __launch_bounds__(256) clip_scale_kernel(float* __restrict__ g, long long n, const double* __restrict__ acc, float clip_norm,
                                                         float* __restrict__ norm_out) {
  const float norm = (float)sqrt(*acc);
  if (blockIdx.x == 0 && threadIdx.x == 0 && norm_out) *norm_out = norm;
  const float scale = clip_norm / fmaxf(norm, clip_norm);
  if (scale == 1.0f) return;
  for (long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * 4; i < n; i += (long long)gridDim.x * blockDim.x * 4) {
    if (i + 4 <= n) {
      float4 v = *reinterpret_cast<float4*>(g + i);
      v.x *= scale; v.y *= scale; v.z *= scale; v.w *= scale;
      *reinterpret_cast<float4*>(g + i) = v;
    } else {
      for (long long j = i; j < n; ++j) g[j] *= scale;
    }
  }
}

}  // namespace mb

using namespace mb;

extern "C" int merlot_clip_by_global_norm(float* g, long long n, float clip_norm, double* scratch_f64, float* norm_out, void* stream_) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
  MB_REQUIRE(g && scratch_f64, MERLOT_EINVAL, "clip_by_global_norm: null pointer");
  MB_REQUIRE(clip_norm > 0.f && ((uintptr_t)g % 16) == 0, MERLOT_EINVAL, "clip_by_global_norm: clip_norm must be > 0 and g 16-byte aligned");
  if (n <= 0) return MERLOT_OK;
  MB_CHECK_CUDA(cudaMemsetAsync(scratch_f64, 0, sizeof(double), st));
  const int grid = device_sms() * 8;
  sumsq_kernel<<<grid, 256, 0, st>>>(g, n, scratch_f64);
  MB_CHECK_LAUNCH();
  clip_scale_kernel<<<grid, 256, 0, st>>>(g, n, scratch_f64, clip_norm, norm_out);
  MB_CHECK_LAUNCH();
  return MERLOT_OK;
}


extern "C" int merlot_adamw_step(const merlot_adamw_t* d, void* stream_) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
  MB_REQUIRE(d && d->p && d->g && d->m && d->v, MERLOT_EINVAL, "adamw_step: null pointer");
  MB_REQUIRE(((uintptr_t)d->p % 16) == 0 && ((uintptr_t)d->g % 16) == 0 && ((uintptr_t)d->m % 16) == 0 &&
                 ((uintptr_t)d->v % 16) == 0 && (!d->p_bf16 || ((uintptr_t)d->p_bf16 % 16) == 0),
             MERLOT_ESHAPE, "adamw_step: buffers must be 16-byte aligned (pad each group to a multiple of 8 elements)");
  if (d->n <= 0) return MERLOT_OK;
  AdamDev a;
  a.p = d->p; a.g = d->g; a.m = (bf16*)d->m; a.v = (bf16*)d->v; a.p_bf16 = (bf16*)d->p_bf16; a.n = d->n;
  a.b1 = d->beta1; a.omb1 = d->one_minus_beta1; a.b2 = d->beta2; a.omb2 = d->one_minus_beta2;
  a.eps = d->epsilon; a.lr_t = d->lr_t; a.wd = d->weight_decay; a.grad_scale = d->grad_scale; a.zero_grad = d->zero_grad;
  adamw_kernel<<<(unsigned)ceil_div_ll(ceil_div_ll(d->n, 8), 256), 256, 0, st>>>(a);
  MB_CHECK_LAUNCH();
  return MERLOT_OK;
}
