// K13: the hybrid ResNet-lite stem (utils/vision_transformer.py:8-170; SURVEY.md 8(f) next-row 1,
// Appendix D).  Every convolution is a K1 GEMM: 1x1 convs read the NHWC activation matrix [N*h*w, C] as it is, 3x3
// convs go through an im2col matrix whose columns are ordered (ky, kx, c) like the flattened HWIO kernel.  This file
// holds what sits between the GEMMs:
//   ws_kernel         weight standardisation (vision_transformer.py:56-60): per OUTPUT channel over (kh, kw, cin), biased
//                     variance, eps 1e-5, fp32 -> bf16 GEMM operand [K_pad, cout]
//   im2col3x3_*       3x3 taps with one ring of zero padding, stride 1 (SAME) or 2 (fixed_padding :8-19 + VALID); the
//                     stride-2 first conv reads the image and subtracts 0.5 (:193) BEFORE the padding zeros
//   gn_stats / apply  batch_norm_relu (:22-27) = GroupNorm(32 groups, eps 1e-4) with the ONE-PASS moments of
//                     utils/model_utils.py:196-201 (mean = sum/n, var = sum(x^2)/n - mean^2), gamma/beta per channel, bf16
//                     out, optional ReLU, optional `relu(out + shortcut)` (bottleneck_block :96)
//   avgpool2          tf.nn.avg_pool2d(ksize 2, strides 2, SAME) (:81,93,159): bottom/right padding not counted
// The second half of the file holds the gradient of the same pieces (GroupNorm/ReLU/shortcut, avg-pool, col2im, weight
// standardisation); HybridStem.backward (stem.py) walks the forward tape and calls them.
#include "host_common.h"
#include "ptx.cuh"

namespace mb {

// Weight standardisation, forward and backward.  A block of WS_WARPS warps owns 32 neighbouring output channels: lane = channel
// (every load is one coalesced 128-byte row segment), the warps split the rows (kh, kw, cin) and meet in shared memory once
// per moment.  History: one THREAD per channel (64..1024 threads in all, a serial loop over up to 2304 rows: 83 us per launch,
// 107 launches per step) -> one warp per channel (19 us, but 32 memory wavefronts per load: lanes on different rows) -> this.
constexpr int WS_CH = 32;    // channels per block
constexpr int WS_WARPS = 32;  // row lanes (1024 threads: the loops over up to 2304 rows are latency chains, 374 us at 8 warps)
__device__ __forceinline__ float ws_block_sum(float v, float (*red)[WS_CH], int warp, int lane) {
  __syncthreads();  // the previous use of `red` is over
  red[warp][lane] = v;
  __syncthreads();
  float t = 0.f;
#pragma unroll
  for (int k = 0; k < WS_WARPS; ++k) t += red[k][lane];
  return t;
}
__device__ __forceinline__ void ws_channels(const float* __restrict__ w, int rows, int rows_pad, int cout, bf16* __restrict__ out, int c0) {
  __shared__ float red[WS_WARPS][WS_CH];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, c = c0 + lane;
  const bool ok = c < cout;
  float mean = 0.f;
#pragma unroll 8
  for (int r = warp; r < rows; r += WS_WARPS) mean += ok ? w[(size_t)r * cout + c] : 0.f;
  mean = ws_block_sum(mean, red, warp, lane) / (float)rows;
  float var = 0.f;
  for (int r = warp; r < rows; r += WS_WARPS) {
    const float d = ok ? w[(size_t)r * cout + c] - mean : 0.f;
    var += d * d;
  }
  var = ws_block_sum(var, red, warp, lane) / (float)rows;
  const float s = rsqrtf(var + 1e-5f);
  if (!ok) return;
  for (int r = warp; r < rows; r += WS_WARPS) out[(size_t)r * cout + c] = __float2bfloat16_rn((w[(size_t)r * cout + c] - mean) * s);
  for (int r = rows + warp; r < rows_pad; r += WS_WARPS) out[(size_t)r * cout + c] = __float2bfloat16_rn(0.f);
}
__global__ void __launch_bounds__(32 * WS_WARPS) ws_kernel(const float* __restrict__ w, int rows, int rows_pad, int cout, bf16* __restrict__ out) {
  ws_channels(w, rows, rows_pad, cout, out, blockIdx.x * WS_CH);
}
// Every conv kernel of the stem in ONE launch (the operands depend on the parameters only): block b serves the item whose
// [block0, next block0) range holds it.
struct WsItem {  // == merlot_ws_item_t
  const float* w; void* out; const float* dws; float* dw;
  int rows, rows_pad, cout, ld_dws, block0, pad_;
};
__device__ __forceinline__ int ws_find_item(const WsItem* __restrict__ items, int n_items) {
  int lo = 0, hi = n_items - 1;  // last item whose block0 <= blockIdx.x (block0 is non-decreasing, item 0 starts at 0)
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (items[mid].block0 <= (int)blockIdx.x) lo = mid; else hi = mid - 1;
  }
  return lo;
}
__global__ void __launch_bounds__(32 * WS_WARPS) ws_multi_kernel(const WsItem* __restrict__ items, int n_items) {
  const WsItem q = items[ws_find_item(items, n_items)];
  ws_channels(q.w, q.rows, q.rows_pad, q.cout, reinterpret_cast<bf16*>(q.out), ((int)blockIdx.x - q.block0) * WS_CH);
}

// C % 8 == 0: one thread per (output pixel, tap, 8 channels)
__global__ void __launch_bounds__(256) im2col3x3_vec_kernel(const bf16* __restrict__ x, int N, int h, int w, int C, int stride, int ho,
                                                            int wo, bf16* __restrict__ out, int ld, long long total) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int c8n = C >> 3;
  const int c8 = (int)(idx % c8n);
  const int tap = (int)((idx / c8n) % 9);
  const long long row = idx / (9LL * c8n);
  const int ox = (int)(row % wo), oy = (int)((row / wo) % ho), n = (int)(row / ((long long)wo * ho));
  const int iy = oy * stride + tap / 3 - 1, ix = ox * stride + tap % 3 - 1;
  uint4 v = make_uint4(0u, 0u, 0u, 0u);
  if (iy >= 0 && iy < h && ix >= 0 && ix < w)
    v = *reinterpret_cast<const uint4*>(x + (((size_t)n * h + iy) * w + ix) * C + c8 * 8);
  *reinterpret_cast<uint4*>(out + (size_t)row * ld + tap * C + c8 * 8) = v;
}

// any C (the 3-channel image): one thread per (output pixel, column); columns [9C, ld) are zero padding for the GEMM's K
__global__ void __launch_bounds__(256) im2col3x3_scalar_kernel(const bf16* __restrict__ x, int N, int h, int w, int C, int stride, int ho,
                                                               int wo, bf16* __restrict__ out, int ld, int sub_half, long long total) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int col = (int)(idx % ld);
  const long long row = idx / ld;
  float v = 0.f;
  if (col < 9 * C) {
    const int tap = col / C, c = col % C;
    const int ox = (int)(row % wo), oy = (int)((row / wo) % ho), n = (int)(row / ((long long)wo * ho));
    const int iy = oy * stride + tap / 3 - 1, ix = ox * stride + tap % 3 - 1;
    if (iy >= 0 && iy < h && ix >= 0 && ix < w) {
      v = __bfloat162float(x[(((size_t)n * h + iy) * w + ix) * C + c]);
      if (sub_half) v -= 0.5f;  // img_norm = image - 0.5 (vision_transformer.py:193); the padding ring stays 0
    }
  }
  out[(size_t)row * ld + col] = __float2bfloat16_rn(v);
}

// per (sample, group): sum and sum of squares over (h*w, channels of the group).  grid (slabs, N); stats must be zero on entry.
__global__ void __launch_bounds__(256) gn_stats_kernel(const bf16* __restrict__ x, int HW, int C, int groups, int rows_per_block,
                                                       float* __restrict__ stats) {
  extern __shared__ float acc[];  // [groups][2]
  const int n = blockIdx.y;
  for (int i = threadIdx.x; i < 2 * groups; i += blockDim.x) acc[i] = 0.f;
  __syncthreads();
  const int c8n = C >> 3;
  const int lanes = blockDim.x / c8n > 0 ? blockDim.x / c8n : 1;  // rows processed in parallel
  const int c8 = threadIdx.x % c8n, rl = threadIdx.x / c8n;
  const int r0 = blockIdx.x * rows_per_block;
  const int r1 = min(HW, r0 + rows_per_block);
  float s[8], q[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) { s[i] = 0.f; q[i] = 0.f; }
  if (rl < lanes && c8 < c8n) {
    for (int r = r0 + rl; r < r1; r += lanes) {
      const uint4 u = *reinterpret_cast<const uint4*>(x + ((size_t)n * HW + r) * C + c8 * 8);
      const uint32_t wv[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float2 f = unpack_bf16x2(wv[i]);
        s[2 * i] += f.x; q[2 * i] += f.x * f.x;
        s[2 * i + 1] += f.y; q[2 * i + 1] += f.y * f.y;
      }
    }
    const int cg = C / groups;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int g = (c8 * 8 + i) / cg;
      atomicAdd(&acc[2 * g], s[i]);
      atomicAdd(&acc[2 * g + 1], q[i]);
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 2 * groups; i += blockDim.x) atomicAdd(&stats[(size_t)n * 2 * groups + i], acc[i]);
}

__global__ void __launch_bounds__(256) gn_apply_kernel(const bf16* __restrict__ x, const float* __restrict__ stats,
                                                       const float* __restrict__ gamma, const float* __restrict__ beta,
                                                       const bf16* __restrict__ shortcut, bf16* __restrict__ y, int HW, int C, int groups,
                                                       float eps, int relu, long long total) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int c8n = C >> 3;
  const int c8 = (int)(idx % c8n);
  const long long row = idx / c8n;
  const int n = (int)(row / HW);
  const int cg = C / groups;
  const float inv_cnt = 1.0f / ((float)HW * (float)cg);
  const uint4 u = *reinterpret_cast<const uint4*>(x + (size_t)row * C + c8 * 8);
  const uint32_t wv[4] = {u.x, u.y, u.z, u.w};
  float v[8];
#pragma unroll
  for (int i = 0; i < 4; ++i) { const float2 f = unpack_bf16x2(wv[i]); v[2 * i] = f.x; v[2 * i + 1] = f.y; }
  float sc[8];
  if (shortcut != nullptr) {
    const uint4 su = *reinterpret_cast<const uint4*>(shortcut + (size_t)row * C + c8 * 8);
    const uint32_t sw[4] = {su.x, su.y, su.z, su.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) { const float2 f = unpack_bf16x2(sw[i]); sc[2 * i] = f.x; sc[2 * i + 1] = f.y; }
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int c = c8 * 8 + i;
    const int g = c / cg;
    const float mean = stats[((size_t)n * groups + g) * 2] * inv_cnt;
    const float var = stats[((size_t)n * groups + g) * 2 + 1] * inv_cnt - mean * mean;  // one-pass moments (model_utils.py:196-201)
    float o = (v[i] - mean) * rsqrtf(var + eps) * gamma[c] + beta[c];
    if (shortcut != nullptr) o = __bfloat162float(__float2bfloat16_rn(o)) + sc[i];  // bf16 tensor + bf16 tensor (:96)
    if (relu) o = fmaxf(o, 0.f);
    v[i] = o;
  }
  *reinterpret_cast<uint4*>(y + (size_t)row * C + c8 * 8) =
      make_uint4(pack_bf16x2(v[0], v[1]), pack_bf16x2(v[2], v[3]), pack_bf16x2(v[4], v[5]), pack_bf16x2(v[6], v[7]));
}

__global__ void __launch_bounds__(256) avgpool2_kernel(const bf16* __restrict__ x, int N, int h, int w, int C, int ho, int wo,
                                                       bf16* __restrict__ y, long long total) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int c8n = C >> 3;
  const int c8 = (int)(idx % c8n);
  const long long row = idx / c8n;
  const int ox = (int)(row % wo), oy = (int)((row / wo) % ho), n = (int)(row / ((long long)wo * ho));
  float a[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) a[i] = 0.f;
  int cnt = 0;
  for (int dy = 0; dy < 2; ++dy)
    for (int dx = 0; dx < 2; ++dx) {
      const int iy = oy * 2 + dy, ix = ox * 2 + dx;
      if (iy < h && ix < w) {
        const uint4 u = *reinterpret_cast<const uint4*>(x + (((size_t)n * h + iy) * w + ix) * C + c8 * 8);
        const uint32_t wv[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) { const float2 f = unpack_bf16x2(wv[i]); a[2 * i] += f.x; a[2 * i + 1] += f.y; }
        ++cnt;
      }
    }
  const float inv = 1.0f / (float)cnt;
  *reinterpret_cast<uint4*>(y + (size_t)row * C + c8 * 8) =
      make_uint4(pack_bf16x2(a[0] * inv, a[1] * inv), pack_bf16x2(a[2] * inv, a[3] * inv), pack_bf16x2(a[4] * inv, a[5] * inv),
                 pack_bf16x2(a[6] * inv, a[7] * inv));
}

// ---------------------------------------------------------------------------------------------------------------------
// backward pieces (gradient of the same graph; vision_transformer.py has no explicit backward -- tf.gradients derives it)
// ---------------------------------------------------------------------------------------------------------------------
// GroupNorm(+ReLU / +shortcut) backward, pass 1: with g = dy * [y > 0] (when relu) and xhat = (x - mean) * rstd,
//   red[n][grp] += { sum g*gamma, sum g*gamma*xhat }   (group sums for dx),   dgamma[c] += sum g*xhat,   dbeta[c] += sum g
__global__ void __launch_bounds__(256) gn_bwd_reduce_kernel(const bf16* __restrict__ dy, const bf16* __restrict__ x,
                                                            const bf16* __restrict__ y, const float* __restrict__ stats,
                                                            const float* __restrict__ gamma, int HW, int C, int groups, float eps,
                                                            int relu, int rows_per_block, float* __restrict__ red,
                                                            float* __restrict__ dgamma, float* __restrict__ dbeta) {
  extern __shared__ float acc[];  // [groups][2] group sums, then [C][2] dgamma / dbeta of this block
  float* cacc = acc + 2 * groups;
  const int n = blockIdx.y;
  for (int i = threadIdx.x; i < 2 * groups + 2 * C; i += blockDim.x) acc[i] = 0.f;
  __syncthreads();
  const int c8n = C >> 3;
  const int lanes = blockDim.x / c8n > 0 ? blockDim.x / c8n : 1;
  const int c8 = threadIdx.x % c8n, rl = threadIdx.x / c8n;
  const int r0 = blockIdx.x * rows_per_block;
  const int r1 = min(HW, r0 + rows_per_block);
  const int cg = C / groups;
  const float inv_cnt = 1.0f / ((float)HW * (float)cg);
  if (rl < lanes) {
    float mean[8], rstd[8], gm[8], s1[8], s2[8], dg[8], db[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int c = c8 * 8 + i;
      const int g = c / cg;
      mean[i] = stats[((size_t)n * groups + g) * 2] * inv_cnt;
      rstd[i] = rsqrtf(stats[((size_t)n * groups + g) * 2 + 1] * inv_cnt - mean[i] * mean[i] + eps);
      gm[i] = gamma[c];
      s1[i] = s2[i] = dg[i] = db[i] = 0.f;
    }
    for (int r = r0 + rl; r < r1; r += lanes) {
      const size_t off = ((size_t)n * HW + r) * C + c8 * 8;
      const uint4 du = *reinterpret_cast<const uint4*>(dy + off);
      const uint4 xu = *reinterpret_cast<const uint4*>(x + off);
      uint4 yu = make_uint4(0u, 0u, 0u, 0u);
      if (relu) yu = *reinterpret_cast<const uint4*>(y + off);
      const uint32_t dw[4] = {du.x, du.y, du.z, du.w}, xw[4] = {xu.x, xu.y, xu.z, xu.w}, yw[4] = {yu.x, yu.y, yu.z, yu.w};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float2 d2 = unpack_bf16x2(dw[i]), x2 = unpack_bf16x2(xw[i]), y2 = unpack_bf16x2(yw[i]);
        const float gv[2] = {(!relu || y2.x > 0.f) ? d2.x : 0.f, (!relu || y2.y > 0.f) ? d2.y : 0.f};
        const float xv[2] = {x2.x, x2.y};
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const int k = 2 * i + j;
          const float xh = (xv[j] - mean[k]) * rstd[k];
          s1[k] += gv[j] * gm[k];
          s2[k] += gv[j] * gm[k] * xh;
          dg[k] += gv[j] * xh;
          db[k] += gv[j];
        }
      }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int c = c8 * 8 + i;
      const int g = c / cg;
      atomicAdd(&acc[2 * g], s1[i]);
      atomicAdd(&acc[2 * g + 1], s2[i]);
      atomicAdd(&cacc[2 * c], dg[i]);  // shared memory first: ONE global reduction per channel and block (every thread used to
      atomicAdd(&cacc[2 * c + 1], db[i]);  // add to the same C addresses in global memory: 142 us per launch at C = 64)
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 2 * groups; i += blockDim.x) atomicAdd(&red[(size_t)n * 2 * groups + i], acc[i]);
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    atomicAdd(&dgamma[c], cacc[2 * c]);
    atomicAdd(&dbeta[c], cacc[2 * c + 1]);
  }
}

// pass 2: dx = rstd * (g*gamma - S1/cnt - xhat * S2/cnt);  dshortcut = g (the residual branch sees the masked gradient)
__global__ void __launch_bounds__(256) gn_bwd_apply_kernel(const bf16* __restrict__ dy, const bf16* __restrict__ x,
                                                           const bf16* __restrict__ y, const float* __restrict__ stats,
                                                           const float* __restrict__ red, const float* __restrict__ gamma,
                                                           bf16* __restrict__ dx, bf16* __restrict__ dshortcut, int HW, int C, int groups,
                                                           float eps, int relu, long long total) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int c8n = C >> 3;
  const int c8 = (int)(idx % c8n);
  const long long row = idx / c8n;
  const int n = (int)(row / HW);
  const int cg = C / groups;
  const float inv_cnt = 1.0f / ((float)HW * (float)cg);
  const size_t off = (size_t)row * C + c8 * 8;
  const uint4 du = *reinterpret_cast<const uint4*>(dy + off);
  const uint4 xu = *reinterpret_cast<const uint4*>(x + off);
  uint4 yu = make_uint4(0u, 0u, 0u, 0u);
  if (relu) yu = *reinterpret_cast<const uint4*>(y + off);
  const uint32_t dw[4] = {du.x, du.y, du.z, du.w}, xw[4] = {xu.x, xu.y, xu.z, xu.w}, yw[4] = {yu.x, yu.y, yu.z, yu.w};
  float o[8], gsc[8];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 d2 = unpack_bf16x2(dw[i]), x2 = unpack_bf16x2(xw[i]), y2 = unpack_bf16x2(yw[i]);
    const float gv[2] = {(!relu || y2.x > 0.f) ? d2.x : 0.f, (!relu || y2.y > 0.f) ? d2.y : 0.f};
    const float xv[2] = {x2.x, x2.y};
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int k = 2 * i + j;
      const int c = c8 * 8 + k;
      const int g = c / cg;
      const float mean = stats[((size_t)n * groups + g) * 2] * inv_cnt;
      const float rstd = rsqrtf(stats[((size_t)n * groups + g) * 2 + 1] * inv_cnt - mean * mean + eps);
      const float xh = (xv[j] - mean) * rstd;
      const float S1 = red[((size_t)n * groups + g) * 2] * inv_cnt, S2 = red[((size_t)n * groups + g) * 2 + 1] * inv_cnt;
      o[k] = rstd * (gv[j] * gamma[c] - S1 - xh * S2);
      gsc[k] = gv[j];
    }
  }
  *reinterpret_cast<uint4*>(dx + off) =
      make_uint4(pack_bf16x2(o[0], o[1]), pack_bf16x2(o[2], o[3]), pack_bf16x2(o[4], o[5]), pack_bf16x2(o[6], o[7]));
  if (dshortcut != nullptr)
    *reinterpret_cast<uint4*>(dshortcut + off) =
        make_uint4(pack_bf16x2(gsc[0], gsc[1]), pack_bf16x2(gsc[2], gsc[3]), pack_bf16x2(gsc[4], gsc[5]), pack_bf16x2(gsc[6], gsc[7]));
}

// avg-pool backward: every input pixel receives dy / (number of valid pixels in its window)
__global__ void __launch_bounds__(256) avgpool2_bwd_kernel(const bf16* __restrict__ dy, int N, int h, int w, int C, int ho, int wo,
                                                           bf16* __restrict__ dx, long long total) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int c8n = C >> 3;
  const int c8 = (int)(idx % c8n);
  const long long row = idx / c8n;
  const int ix = (int)(row % w), iy = (int)((row / w) % h), n = (int)(row / ((long long)w * h));
  const int oy = iy >> 1, ox = ix >> 1;
  const int cnt = ((oy * 2 + 1 < h) ? 2 : 1) * ((ox * 2 + 1 < w) ? 2 : 1);
  const float inv = 1.0f / (float)cnt;
  const uint4 u = *reinterpret_cast<const uint4*>(dy + (((size_t)n * ho + oy) * wo + ox) * C + c8 * 8);
  const uint32_t wv[4] = {u.x, u.y, u.z, u.w};
  float a[8];
#pragma unroll
  for (int i = 0; i < 4; ++i) { const float2 f = unpack_bf16x2(wv[i]); a[2 * i] = f.x * inv; a[2 * i + 1] = f.y * inv; }
  *reinterpret_cast<uint4*>(dx + (size_t)row * C + c8 * 8) =
      make_uint4(pack_bf16x2(a[0], a[1]), pack_bf16x2(a[2], a[3]), pack_bf16x2(a[4], a[5]), pack_bf16x2(a[6], a[7]));
}

// col2im for the 3x3 taps: dx[n, iy, ix, :] = sum over taps of dcol[row(oy, ox), tap*C : tap*C + C] with oy*stride + ky - 1 == iy
__global__ void __launch_bounds__(256) col2im3x3_kernel(const bf16* __restrict__ dcol, int N, int h, int w, int C, int stride, int ho,
                                                        int wo, int ld, bf16* __restrict__ dx, long long total) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int c8n = C >> 3;
  const int c8 = (int)(idx % c8n);
  const long long pix = idx / c8n;
  const int ix = (int)(pix % w), iy = (int)((pix / w) % h), n = (int)(pix / ((long long)w * h));
  float a[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) a[i] = 0.f;
  for (int ky = 0; ky < 3; ++ky) {
    const int ty = iy - ky + 1;
    if (ty < 0 || ty % stride != 0) continue;
    const int oy = ty / stride;
    if (oy >= ho) continue;
    for (int kx = 0; kx < 3; ++kx) {
      const int tx = ix - kx + 1;
      if (tx < 0 || tx % stride != 0) continue;
      const int ox = tx / stride;
      if (ox >= wo) continue;
      const uint4 u = *reinterpret_cast<const uint4*>(dcol + (((size_t)n * ho + oy) * wo + ox) * ld + (ky * 3 + kx) * C + c8 * 8);
      const uint32_t wv[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
      for (int i = 0; i < 4; ++i) { const float2 f = unpack_bf16x2(wv[i]); a[2 * i] += f.x; a[2 * i + 1] += f.y; }
    }
  }
  *reinterpret_cast<uint4*>(dx + (size_t)pix * C + c8 * 8) =
      make_uint4(pack_bf16x2(a[0], a[1]), pack_bf16x2(a[2], a[3]), pack_bf16x2(a[4], a[5]), pack_bf16x2(a[6], a[7]));
}

// weight-standardisation backward, per output channel: what = (w - mean) * rstd,
//   dw += rstd * (dws - mean_r(dws) - what * mean_r(dws * what))
__device__ __forceinline__ void ws_bwd_channels(const float* __restrict__ dws, int ld_dws, const float* __restrict__ w, int rows, int cout,
                                                float* __restrict__ dw, int c0) {
  __shared__ float red[WS_WARPS][WS_CH];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, c = c0 + lane;  // same mapping as ws_channels
  const bool ok = c < cout;
  float mean = 0.f;
#pragma unroll 8
  for (int r = warp; r < rows; r += WS_WARPS) mean += ok ? w[(size_t)r * cout + c] : 0.f;
  mean = ws_block_sum(mean, red, warp, lane) / (float)rows;
  float var = 0.f;
  for (int r = warp; r < rows; r += WS_WARPS) { const float d = ok ? w[(size_t)r * cout + c] - mean : 0.f; var += d * d; }
  var = ws_block_sum(var, red, warp, lane) / (float)rows;
  const float rstd = rsqrtf(var + 1e-5f);
  float m1 = 0.f, m2 = 0.f;
  for (int r = warp; r < rows; r += WS_WARPS) {
    const float g = ok ? dws[(size_t)r * ld_dws + c] : 0.f;
    m1 += g;
    m2 += ok ? g * (w[(size_t)r * cout + c] - mean) * rstd : 0.f;
  }
  m1 = ws_block_sum(m1, red, warp, lane) / (float)rows;
  m2 = ws_block_sum(m2, red, warp, lane) / (float)rows;
  if (!ok) return;
  for (int r = warp; r < rows; r += WS_WARPS) {
    const float wh = (w[(size_t)r * cout + c] - mean) * rstd;
    dw[(size_t)r * cout + c] += rstd * (dws[(size_t)r * ld_dws + c] - m1 - wh * m2);
  }
}
__global__ void __launch_bounds__(32 * WS_WARPS) ws_bwd_kernel(const float* __restrict__ dws, int ld_dws, const float* __restrict__ w, int rows,
                                                               int cout, float* __restrict__ dw) {
  ws_bwd_channels(dws, ld_dws, w, rows, cout, dw, blockIdx.x * WS_CH);
}
__global__ void __launch_bounds__(32 * WS_WARPS) ws_bwd_multi_kernel(const WsItem* __restrict__ items, int n_items) {
  const WsItem q = items[ws_find_item(items, n_items)];
  ws_bwd_channels(q.dws, q.ld_dws, q.w, q.rows, q.cout, q.dw, ((int)blockIdx.x - q.block0) * WS_CH);
}

__global__ void __launch_bounds__(256) add_bf16_kernel(const bf16* __restrict__ a, const bf16* __restrict__ b, bf16* __restrict__ out,
                                                       long long n8) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n8) return;
  const uint4 ua = *reinterpret_cast<const uint4*>(a + idx * 8), ub = *reinterpret_cast<const uint4*>(b + idx * 8);
  const uint32_t aw[4] = {ua.x, ua.y, ua.z, ua.w}, bw[4] = {ub.x, ub.y, ub.z, ub.w};
  uint32_t o[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 fa = unpack_bf16x2(aw[i]), fb = unpack_bf16x2(bw[i]);
    o[i] = pack_bf16x2(fa.x + fb.x, fa.y + fb.y);
  }
  *reinterpret_cast<uint4*>(out + idx * 8) = make_uint4(o[0], o[1], o[2], o[3]);
}

}  // namespace mb

using namespace mb;

#define GRID1D(n) (unsigned)ceil_div_ll((n), 256), 256, 0, st

extern "C" int merlot_ws_weights(const float* w, int rows, int rows_pad, int cout, void* out_bf16, void* stream_) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
  MB_REQUIRE(w && out_bf16, MERLOT_EINVAL, "ws_weights: null pointer");
  MB_REQUIRE(rows > 0 && rows_pad >= rows && cout > 0, MERLOT_ESHAPE, "ws_weights: bad shape rows=%d rows_pad=%d cout=%d", rows, rows_pad, cout);
  ws_kernel<<<(unsigned)ceil_div(cout, WS_CH), 32 * WS_WARPS, 0, st>>>(w, rows, rows_pad, cout, (bf16*)out_bf16);
  MB_CHECK_LAUNCH();
  return MERLOT_OK;
}

extern "C" int merlot_im2col3x3(const void* x_bf16, int N, int h, int w, int C, int stride, int sub_half, void* out_bf16, int ld,
                                void* stream_) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
  MB_REQUIRE(x_bf16 && out_bf16, MERLOT_EINVAL, "im2col3x3: null pointer");
  MB_REQUIRE(N > 0 && h > 0 && w > 0 && C > 0 && (stride == 1 || stride == 2), MERLOT_ESHAPE, "im2col3x3: bad shape / stride %d", stride);
  MB_REQUIRE(ld >= 9 * C && ld % 8 == 0, MERLOT_ESHAPE, "im2col3x3: ld=%d must be >= 9*C and a multiple of 8", ld);
  const int ho = (h + 2 - 3) / stride + 1, wo = (w + 2 - 3) / stride + 1;
  const long long rows = (long long)N * ho * wo;
  if (C % 8 == 0 && ld == 9 * C && !sub_half) {
    const long long total = rows * 9 * (C / 8);
    im2col3x3_vec_kernel<<<GRID1D(total)>>>((const bf16*)x_bf16, N, h, w, C, stride, ho, wo, (bf16*)out_bf16, ld, total);
  } else {
    const long long total = rows * ld;
    im2col3x3_scalar_kernel<<<GRID1D(total)>>>((const bf16*)x_bf16, N, h, w, C, stride, ho, wo, (bf16*)out_bf16, ld, sub_half, total);
  }
  MB_CHECK_LAUNCH();
  return MERLOT_OK;
}

extern "C" int merlot_group_norm_fwd(const void* x_bf16, const float* gamma, const float* beta, const void* shortcut_bf16, void* y_bf16,
                                     float* stats, int N, int HW, int C, int groups, float eps, int relu, void* stream_) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
  MB_REQUIRE(x_bf16 && gamma && beta && y_bf16 && stats, MERLOT_EINVAL, "group_norm_fwd: null pointer");
  MB_REQUIRE(groups > 0 && C % groups == 0, MERLOT_ESHAPE, "group_norm_fwd: %d channels is not commensurate with %d groups", C, groups);
  MB_REQUIRE(C % 8 == 0 && C / 8 <= 256 && groups <= 1024, MERLOT_ESHAPE, "group_norm_fwd: C must be a multiple of 8 and <= 2048 (got %d)", C);
  if (N == 0 || HW == 0) return MERLOT_OK;
  MB_CHECK_CUDA(cudaMemsetAsync(stats, 0, sizeof(float) * 2 * (size_t)groups * N, st));
  const int lanes = 256 / (C / 8);
  int rows_per_block = lanes * 32;  // every thread reduces ~32 rows before touching shared memory
  if (rows_per_block > HW) rows_per_block = HW;
  dim3 grid((unsigned)ceil_div(HW, rows_per_block), (unsigned)N);
  gn_stats_kernel<<<grid, 256, 2 * groups * sizeof(float), st>>>((const bf16*)x_bf16, HW, C, groups, rows_per_block, stats);
  MB_CHECK_LAUNCH();
  const long long total = (long long)N * HW * (C / 8);
  gn_apply_kernel<<<GRID1D(total)>>>((const bf16*)x_bf16, stats, gamma, beta, (const bf16*)shortcut_bf16, (bf16*)y_bf16, HW, C, groups,
                                     eps, relu, total);
  MB_CHECK_LAUNCH();
  return MERLOT_OK;
}

extern "C" int merlot_avgpool2_same(const void* x_bf16, int N, int h, int w, int C, void* y_bf16, void* stream_) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
  MB_REQUIRE(x_bf16 && y_bf16, MERLOT_EINVAL, "avgpool2_same: null pointer");
  MB_REQUIRE(C % 8 == 0 && N > 0 && h > 0 && w > 0, MERLOT_ESHAPE, "avgpool2_same: C must be a multiple of 8 (got %d)", C);
  const int ho = (h + 1) / 2, wo = (w + 1) / 2;
  const long long total = (long long)N * ho * wo * (C / 8);
  avgpool2_kernel<<<GRID1D(total)>>>((const bf16*)x_bf16, N, h, w, C, ho, wo, (bf16*)y_bf16, total);
  MB_CHECK_LAUNCH();
  return MERLOT_OK;
}

extern "C" int merlot_group_norm_bwd(const void* dy_bf16, const void* x_bf16, const void* y_bf16, const float* stats, const float* gamma,
                                     void* dx_bf16, void* dshortcut_bf16, float* dgamma, float* dbeta, float* red, int N, int HW, int C,
                                     int groups, float eps, int relu, void* stream_) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
  MB_REQUIRE(dy_bf16 && x_bf16 && stats && gamma && dx_bf16 && dgamma && dbeta && red, MERLOT_EINVAL, "group_norm_bwd: null pointer");
  MB_REQUIRE(!relu || y_bf16, MERLOT_EINVAL, "group_norm_bwd: the ReLU mask needs the forward output y");
  MB_REQUIRE(groups > 0 && C % groups == 0 && C % 8 == 0 && C / 8 <= 256, MERLOT_ESHAPE, "group_norm_bwd: bad C=%d groups=%d", C, groups);
  if (N == 0 || HW == 0) return MERLOT_OK;
  MB_CHECK_CUDA(cudaMemsetAsync(red, 0, sizeof(float) * 2 * (size_t)groups * N, st));
  const int lanes = 256 / (C / 8);
  int rows_per_block = lanes * 32;
  if (rows_per_block > HW) rows_per_block = HW;
  dim3 grid((unsigned)ceil_div(HW, rows_per_block), (unsigned)N);
  gn_bwd_reduce_kernel<<<grid, 256, (2 * groups + 2 * C) * sizeof(float), st>>>((const bf16*)dy_bf16, (const bf16*)x_bf16, (const bf16*)y_bf16, stats,
                                                                      gamma, HW, C, groups, eps, relu, rows_per_block, red, dgamma, dbeta);
  MB_CHECK_LAUNCH();
  const long long total = (long long)N * HW * (C / 8);
  gn_bwd_apply_kernel<<<GRID1D(total)>>>((const bf16*)dy_bf16, (const bf16*)x_bf16, (const bf16*)y_bf16, stats, red, gamma, (bf16*)dx_bf16,
                                         (bf16*)dshortcut_bf16, HW, C, groups, eps, relu, total);
  MB_CHECK_LAUNCH();
  return MERLOT_OK;
}

extern "C" int merlot_avgpool2_same_bwd(const void* dy_bf16, int N, int h, int w, int C, void* dx_bf16, void* stream_) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
  MB_REQUIRE(dy_bf16 && dx_bf16, MERLOT_EINVAL, "avgpool2_same_bwd: null pointer");
  MB_REQUIRE(C % 8 == 0 && N > 0 && h > 0 && w > 0, MERLOT_ESHAPE, "avgpool2_same_bwd: C must be a multiple of 8 (got %d)", C);
  const long long total = (long long)N * h * w * (C / 8);
  avgpool2_bwd_kernel<<<GRID1D(total)>>>((const bf16*)dy_bf16, N, h, w, C, (h + 1) / 2, (w + 1) / 2, (bf16*)dx_bf16, total);
  MB_CHECK_LAUNCH();
  return MERLOT_OK;
}

extern "C" int merlot_col2im3x3(const void* dcol_bf16, int N, int h, int w, int C, int stride, int ld, void* dx_bf16, void* stream_) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
  MB_REQUIRE(dcol_bf16 && dx_bf16, MERLOT_EINVAL, "col2im3x3: null pointer");
  MB_REQUIRE(C % 8 == 0 && ld >= 9 * C && ld % 8 == 0 && (stride == 1 || stride == 2), MERLOT_ESHAPE,
             "col2im3x3: C %% 8 == 0, ld >= 9*C, ld %% 8 == 0 and stride 1 or 2 required (C=%d ld=%d stride=%d)", C, ld, stride);
  const int ho = (h + 2 - 3) / stride + 1, wo = (w + 2 - 3) / stride + 1;
  const long long total = (long long)N * h * w * (C / 8);
  col2im3x3_kernel<<<GRID1D(total)>>>((const bf16*)dcol_bf16, N, h, w, C, stride, ho, wo, ld, (bf16*)dx_bf16, total);
  MB_CHECK_LAUNCH();
  return MERLOT_OK;
}

extern "C" int merlot_ws_weights_bwd(const float* dws, int ld_dws, const float* w, int rows, int cout, float* dw, void* stream_) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
  MB_REQUIRE(dws && w && dw, MERLOT_EINVAL, "ws_weights_bwd: null pointer");
  MB_REQUIRE(rows > 0 && cout > 0 && ld_dws >= cout, MERLOT_ESHAPE, "ws_weights_bwd: bad shape rows=%d cout=%d ld=%d", rows, cout, ld_dws);
  ws_bwd_kernel<<<(unsigned)ceil_div(cout, WS_CH), 32 * WS_WARPS, 0, st>>>(dws, ld_dws, w, rows, cout, dw);
  MB_CHECK_LAUNCH();
  return MERLOT_OK;
}

static_assert(sizeof(WsItem) == sizeof(merlot_ws_item_t), "WsItem must mirror merlot_ws_item_t");
extern "C" int merlot_ws_weights_multi(const merlot_ws_item_t* items_dev, int n_items, int n_blocks, void* stream_) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
  MB_REQUIRE(items_dev && n_items > 0 && n_blocks > 0, MERLOT_EINVAL, "ws_weights_multi: empty item table");
  ws_multi_kernel<<<(unsigned)n_blocks, 32 * WS_WARPS, 0, st>>>(reinterpret_cast<const WsItem*>(items_dev), n_items);
  MB_CHECK_LAUNCH();
  return MERLOT_OK;
}

extern "C" int merlot_ws_weights_bwd_multi(const merlot_ws_item_t* items_dev, int n_items, int n_blocks, void* stream_) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
  MB_REQUIRE(items_dev && n_items > 0 && n_blocks > 0, MERLOT_EINVAL, "ws_weights_bwd_multi: empty item table");
  ws_bwd_multi_kernel<<<(unsigned)n_blocks, 32 * WS_WARPS, 0, st>>>(reinterpret_cast<const WsItem*>(items_dev), n_items);
  MB_CHECK_LAUNCH();
  return MERLOT_OK;
}

extern "C" int merlot_add_bf16(const void* a, const void* b, void* out, long long n, void* stream_) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
  MB_REQUIRE(a && b && out, MERLOT_EINVAL, "add_bf16: null pointer");
  MB_REQUIRE(n % 8 == 0, MERLOT_ESHAPE, "add_bf16: n must be a multiple of 8");
  if (n == 0) return MERLOT_OK;
  add_bf16_kernel<<<GRID1D(n / 8)>>>((const bf16*)a, (const bf16*)b, (bf16*)out, n / 8);
  MB_CHECK_LAUNCH();
  return MERLOT_OK;
}
