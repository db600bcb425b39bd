// K5 and friends: HBM-bound row-wise kernels -- LayerNorm fwd/bwd, bias-gradient column sums, dropout mask re-application,
// row gather / scatter-add, GeLU backward, l2-normalise, softmax cross-entropy.  All use 128-bit vectorised, coalesced
// accesses: one warp owns a row, lane i owns the 16-byte chunks {i, i+32, i+64, ...} of that row.
//
// Reference call sites: utils/model_utils.py:113-130 (layer_norm), :313-332 (raw_cross_entropy_with_logits),
// :335-349 (dropout), :225-235 (one_hot_gather); model/modeling.py:43 (l2_normalize), :533-551 (mask_loss).
#include "host_common.h"
#include "ptx.cuh"

namespace mb {

constexpr int LN_MAX_CHUNKS = 4;  // 8 elements per chunk per lane -> H <= 32*8*4 = 1024

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

template <typename T> struct Vec8;
template <> struct Vec8<bf16> {
  static __device__ __forceinline__ void load(const bf16* p, float (&v)[8]) {
    uint4 u = *reinterpret_cast<const uint4*>(p);
    float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), c = unpack_bf16x2(u.z), d = unpack_bf16x2(u.w);
    v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y; v[4] = c.x; v[5] = c.y; v[6] = d.x; v[7] = d.y;
  }
  static __device__ __forceinline__ void store(bf16* p, const float (&v)[8]) {
    *reinterpret_cast<uint4*>(p) =
        make_uint4(pack_bf16x2(v[0], v[1]), pack_bf16x2(v[2], v[3]), pack_bf16x2(v[4], v[5]), pack_bf16x2(v[6], v[7]));
  }
};
template <> struct Vec8<float> {
  static __device__ __forceinline__ void load(const float* p, float (&v)[8]) {
    float4 a = *reinterpret_cast<const float4*>(p), b = *reinterpret_cast<const float4*>(p + 4);
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
  }
  static __device__ __forceinline__ void store(float* p, const float (&v)[8]) {
    *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
    *reinterpret_cast<float4*>(p + 4) = make_float4(v[4], v[5], v[6], v[7]);
  }
};

// destination row of logical row r: rows are grouped (`per` rows per group), groups are `stride` rows apart, + offset.
__device__ __forceinline__ long long remap_row(long long r, int per, int stride, int offset) {
  return per > 0 ? (r / per) * (long long)stride + offset + (r % per) : r;
}

// -----------------------------------------------------------------------------------------------------------------
// LayerNorm forward: y = x*s - mean*s + beta, s = rsqrt(var + eps) * gamma  (utils/model_utils.py:121-127)
// -----------------------------------------------------------------------------------------------------------------
template <typename TI, typename TO>
__global__ void __launch_bounds__(256) ln_fwd_kernel(const TI* __restrict__ x, int ld_x, TO* __restrict__ y, int ld_y,
                                                     const float* __restrict__ gamma, const float* __restrict__ beta,
                                                     float* __restrict__ mean_out, float* __restrict__ rstd_out, long long rows,
                                                     int H, float eps, int map_per, int map_stride, int map_off,
                                                     uint32_t drop_thresh16, float drop_scale, uint64_t seed, uint32_t site) {
  pdl_launch_dependents();
  pdl_wait();
  const int lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int nchunk = H >> 3;
  float v[LN_MAX_CHUNKS][8];
  float sum = 0.f;
#pragma unroll
  for (int j = 0; j < LN_MAX_CHUNKS; ++j) {
    const int c = lane + 32 * j;
    if (c < nchunk) {
      Vec8<TI>::load(x + (size_t)row * ld_x + c * 8, v[j]);
#pragma unroll
      for (int i = 0; i < 8; ++i) sum += v[j][i];
    }
  }
  const float mean = warp_sum(sum) / (float)H;
  float sq = 0.f;
#pragma unroll
  for (int j = 0; j < LN_MAX_CHUNKS; ++j) {
    const int c = lane + 32 * j;
    if (c < nchunk) {
#pragma unroll
      for (int i = 0; i < 8; ++i) { const float d = v[j][i] - mean; sq += d * d; }
    }
  }
  const float var = warp_sum(sq) / (float)H;
  const float rstd = rsqrtf(var + eps);
  if (lane == 0) {
    if (mean_out) mean_out[row] = mean;
    if (rstd_out) rstd_out[row] = rstd;
  }
  const long long orow = remap_row(row, map_per, map_stride, map_off);
#pragma unroll
  for (int j = 0; j < LN_MAX_CHUNKS; ++j) {
    const int c = lane + 32 * j;
    if (c < nchunk) {
      float g[8], b[8], o[8];
      Vec8<float>::load(gamma + c * 8, g);
      Vec8<float>::load(beta + c * 8, b);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float s = rstd * g[i];
        o[i] = v[j][i] * s - mean * s + b[i];
      }
      if (drop_thresh16) {
        const uint64_t lin = (uint64_t)row * (uint64_t)H + (uint64_t)c * 8;
        const uint32_t keep = dropout_keep8(seed, site, lin >> 3, drop_thresh16);
#pragma unroll
        for (int i = 0; i < 8; ++i) o[i] = ((keep >> i) & 1u) ? o[i] * drop_scale : 0.f;
      }
      Vec8<TO>::store(y + (size_t)orow * ld_y + c * 8, o);
    }
  }
}

// -----------------------------------------------------------------------------------------------------------------
// LayerNorm backward.  dx = rstd * (g*dy - mean(g*dy) - xhat * mean(g*dy*xhat)); optional residual gradient add;
// per-block partial dgamma/dbeta -> second kernel accumulates into the gradient buffer.
// -----------------------------------------------------------------------------------------------------------------
template <typename TX, typename TDY, typename TDX>
__global__ void __launch_bounds__(256) ln_bwd_kernel(const TDY* __restrict__ dy, int ld_dy, const TX* __restrict__ x, int ld_x,
                                                     const float* __restrict__ mean, const float* __restrict__ rstd,
                                                     const float* __restrict__ gamma, const TDX* __restrict__ dres, int ld_dres,
                                                     TDX* __restrict__ dx, int ld_dx, float* __restrict__ partial, long long rows,
                                                     int H, int map_per, int map_stride, int map_off, uint32_t drop_thresh16,
                                                     float drop_scale, uint64_t seed, uint32_t site) {
  extern __shared__ float sred[];  // [2][H]
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarp = blockDim.x >> 5;
  const int nchunk = H >> 3;
  for (int i = threadIdx.x; i < 2 * H; i += blockDim.x) sred[i] = 0.f;
  __syncthreads();
  float dg[LN_MAX_CHUNKS][8], db[LN_MAX_CHUNKS][8], g[LN_MAX_CHUNKS][8];
#pragma unroll
  for (int j = 0; j < LN_MAX_CHUNKS; ++j) {
    const int c = lane + 32 * j;
#pragma unroll
    for (int i = 0; i < 8; ++i) { dg[j][i] = 0.f; db[j][i] = 0.f; g[j][i] = 0.f; }
    if (c < nchunk) Vec8<float>::load(gamma + c * 8, g[j]);
  }
  for (long long row = (long long)blockIdx.x * nwarp + warp; row < rows; row += (long long)gridDim.x * nwarp) {
    const long long yrow = remap_row(row, map_per, map_stride, map_off);
    const float mu = mean[row], rs = rstd[row];
    float xh[LN_MAX_CHUNKS][8], gd[LN_MAX_CHUNKS][8];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int j = 0; j < LN_MAX_CHUNKS; ++j) {
      const int c = lane + 32 * j;
      if (c < nchunk) {
        float xv[8], dv[8];
        Vec8<TX>::load(x + (size_t)row * ld_x + c * 8, xv);
        Vec8<TDY>::load(dy + (size_t)yrow * ld_dy + c * 8, dv);
        if (drop_thresh16) {  // dy is the gradient of dropout(LN(x)): re-apply the forward mask
          const uint64_t lin = (uint64_t)row * (uint64_t)H + (uint64_t)c * 8;
          const uint32_t keep = dropout_keep8(seed, site, lin >> 3, drop_thresh16);
#pragma unroll
          for (int i = 0; i < 8; ++i) dv[i] = ((keep >> i) & 1u) ? dv[i] * drop_scale : 0.f;
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          xh[j][i] = (xv[i] - mu) * rs;
          gd[j][i] = g[j][i] * dv[i];
          s1 += gd[j][i];
          s2 += gd[j][i] * xh[j][i];
          dg[j][i] += dv[i] * xh[j][i];
          db[j][i] += dv[i];
        }
      }
    }
    s1 = warp_sum(s1) / (float)H;
    s2 = warp_sum(s2) / (float)H;
#pragma unroll
    for (int j = 0; j < LN_MAX_CHUNKS; ++j) {
      const int c = lane + 32 * j;
      if (c < nchunk) {
        float o[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) o[i] = rs * (gd[j][i] - s1 - xh[j][i] * s2);
        if (dres != nullptr) {
          float r[8];
          Vec8<TDX>::load(dres + (size_t)row * ld_dres + c * 8, r);
#pragma unroll
          for (int i = 0; i < 8; ++i) o[i] += r[i];
        }
        Vec8<TDX>::store(dx + (size_t)row * ld_dx + c * 8, o);
      }
    }
  }
#pragma unroll
  for (int j = 0; j < LN_MAX_CHUNKS; ++j) {
    const int c = lane + 32 * j;
    if (c < nchunk) {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        atomicAdd(&sred[c * 8 + i], dg[j][i]);
        atomicAdd(&sred[H + c * 8 + i], db[j][i]);
      }
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 2 * H; i += blockDim.x) partial[(size_t)blockIdx.x * 2 * H + i] = sred[i];
}

// -----------------------------------------------------------------------------------------------------------------
// Fused bf16 LayerNorm backward for the transformer stacks.  One pass over (dy, x, dres) produces
//   dx = LN'(dy) + dres                                   (the residual-stream gradient)
//   dmask = dropout_bwd(dx)   (optional)                  (A operand of the next dgrad/wgrad GEMMs)
//   partial[block] = { sum dy*xhat, sum dy, sum dmask }   (dgamma, dbeta, and the bias gradient of the next linear)
// x and dy stay packed (bf16x2) in registers between the two sweeps so 2 blocks of 8 warps fit per SM.
// -----------------------------------------------------------------------------------------------------------------
constexpr int LNF_WARPS = 12;  // one block of 12 warps per SM: the column partials meet in smem, one red.add set per block
constexpr int LNF_STAGES = 3;  // rows in flight per warp
// Rows reach the warp through a private ring of LNF_STAGES row slots filled by 1-D bulk copies (cp.async.bulk, completion on
// an mbarrier of the warp): the loads of the next two rows are in the air while a row is reduced, so the per-row chain
// load -> reduce -> store no longer pays the memory latency once per row (it ran at ~2.5 TB/s with register loads).
__device__ __forceinline__ void bulk_load_row(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_dst)),
               "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__host__ __device__ constexpr size_t lnf_smem_bytes(int H) {  // ring [warp][stage][x | dy | dres][H] bf16 (the fp32 column partials reuse it) + barriers
  return (size_t)LNF_WARPS * LNF_STAGES * 3 * H * 2 + (size_t)LNF_WARPS * LNF_STAGES * 8;
}
// one lane: fetch row r (the warp's k-th) into slot k % LNF_STAGES of the warp's ring
__device__ __forceinline__ void lnf_issue(uint8_t* ring, uint64_t* bar, int k, long long r, const bf16* x, const bf16* dy, const bf16* dres, int H) {
  const int s = k % LNF_STAGES;
  const uint32_t row_bytes = (uint32_t)H * 2u;
  uint8_t* slot = ring + (size_t)s * 3 * row_bytes;
  mbar_arrive_expect_tx(&bar[s], (dres != nullptr ? 3u : 2u) * row_bytes);
  bulk_load_row(slot, x + (size_t)r * H, row_bytes, &bar[s]);
  bulk_load_row(slot + row_bytes, dy + (size_t)r * H, row_bytes, &bar[s]);
  if (dres != nullptr) bulk_load_row(slot + 2 * row_bytes, dres + (size_t)r * H, row_bytes, &bar[s]);
}
template <int NCH>  // 16-byte chunks per lane: NCH = ceil(H / 256), H % 8 == 0 (H = 768 -> NCH = 3)
__global__ void __launch_bounds__(32 * LNF_WARPS, 1)
ln_bwd_fused_kernel(const bf16* __restrict__ dy, const bf16* __restrict__ x, const float* __restrict__ mean,
                    const float* __restrict__ rstd, const float* __restrict__ gamma, const bf16* __restrict__ dres,
                    bf16* __restrict__ dx, bf16* __restrict__ dmask, float* __restrict__ out_g, float* __restrict__ out_b,
                    float* __restrict__ out_bias, long long rows, int H, int want_bias,
                    uint32_t drop_thresh16, float drop_scale, uint64_t seed, uint32_t site) {
  extern __shared__ __align__(16) uint8_t lnf_smem[];
  float* sred = reinterpret_cast<float*>(lnf_smem);  // after the row loop: [LNF_WARPS][3][H] column partials (dgamma | dbeta | bias)
  pdl_launch_dependents();
  const int nchunk = H >> 3;
  const float invH = 1.0f / (float)H;
  // warp index through a shuffle + elect.sync: the bulk copies take uniform-register operands (see gemm_kernel.cuh)
  const int lane = threadIdx.x & 31, warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0), nwarp = blockDim.x >> 5;
  const bool leader = elect_one();
  const uint32_t row_bytes = (uint32_t)H * 2u;
  uint8_t* ring = lnf_smem + (size_t)warp * LNF_STAGES * 3 * row_bytes;
  uint64_t* bar = reinterpret_cast<uint64_t*>(lnf_smem + (size_t)LNF_WARPS * LNF_STAGES * 3 * row_bytes) + warp * LNF_STAGES;
  if (leader) {
#pragma unroll
    for (int s = 0; s < LNF_STAGES; ++s) mbar_init(&bar[s], 1);
    fence_barrier_init();
  }
  __syncwarp();
  const long long row0 = (long long)blockIdx.x * nwarp + warp, row_step = (long long)gridDim.x * nwarp;
  const int n_my = row0 < rows ? (int)((rows - row0 + row_step - 1) / row_step) : 0;
  pdl_wait();
  if (leader) {
    for (int k = 0; k < LNF_STAGES && k < n_my; ++k) lnf_issue(ring, bar, k, row0 + (long long)k * row_step, x, dy, dres, H);
  }
  float dg[NCH][8], db[NCH][8], bs[NCH][8];
#pragma unroll
  for (int j = 0; j < NCH; ++j)
#pragma unroll
    for (int i = 0; i < 8; ++i) { dg[j][i] = 0.f; db[j][i] = 0.f; bs[j][i] = 0.f; }
  float mu_n = 0.f, rs_n = 0.f;
  if (n_my > 0) { mu_n = mean[row0]; rs_n = rstd[row0]; }
  int stage = 0;
  uint32_t phase = 0;
  for (int k = 0; k < n_my; ++k) {
    const long long row = row0 + (long long)k * row_step;
    const float mu = mu_n, rs = rs_n;
    if (k + 1 < n_my) { mu_n = mean[row + row_step]; rs_n = rstd[row + row_step]; }
    const uint8_t* slot = ring + (size_t)stage * 3 * row_bytes;
    mbar_wait(&bar[stage], phase);
    uint4 xp[NCH], dp[NCH];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int j = 0; j < NCH; ++j) {
      const int c = (lane + 32 * j) * 8;
      if (lane + 32 * j < nchunk) {
        xp[j] = *reinterpret_cast<const uint4*>(slot + (size_t)c * 2);
        dp[j] = *reinterpret_cast<const uint4*>(slot + row_bytes + (size_t)c * 2);
      }
    }
#pragma unroll
    for (int j = 0; j < NCH; ++j) {
      const int c = (lane + 32 * j) * 8;
      if (lane + 32 * j >= nchunk) continue;
      float g[8];
      Vec8<float>::load(gamma + c, g);
      const uint32_t* xu = reinterpret_cast<const uint32_t*>(&xp[j]);
      const uint32_t* du = reinterpret_cast<const uint32_t*>(&dp[j]);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float2 xv = unpack_bf16x2(xu[i]), dv = unpack_bf16x2(du[i]);
        const float xh0 = (xv.x - mu) * rs, xh1 = (xv.y - mu) * rs;
        const float gd0 = g[2 * i] * dv.x, gd1 = g[2 * i + 1] * dv.y;
        s1 += gd0 + gd1;
        s2 += gd0 * xh0 + gd1 * xh1;
        dg[j][2 * i] += dv.x * xh0; dg[j][2 * i + 1] += dv.y * xh1;
        db[j][2 * i] += dv.x; db[j][2 * i + 1] += dv.y;
      }
    }
    s1 = warp_sum(s1) * invH;
    s2 = warp_sum(s2) * invH;
#pragma unroll
    for (int j = 0; j < NCH; ++j) {
      const int c = (lane + 32 * j) * 8;
      if (lane + 32 * j >= nchunk) continue;
      float g[8], o[8];
      Vec8<float>::load(gamma + c, g);
      const uint32_t* xu = reinterpret_cast<const uint32_t*>(&xp[j]);
      const uint32_t* du = reinterpret_cast<const uint32_t*>(&dp[j]);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float2 xv = unpack_bf16x2(xu[i]), dv = unpack_bf16x2(du[i]);
        o[2 * i] = rs * (g[2 * i] * dv.x - s1 - (xv.x - mu) * rs * s2);
        o[2 * i + 1] = rs * (g[2 * i + 1] * dv.y - s1 - (xv.y - mu) * rs * s2);
      }
      if (dres != nullptr) {
        float r[8];
        Vec8<bf16>::load(reinterpret_cast<const bf16*>(slot + 2 * row_bytes) + c, r);
#pragma unroll
        for (int i = 0; i < 8; ++i) o[i] += r[i];
      }
      Vec8<bf16>::store(dx + (size_t)row * H + c, o);
      if (want_bias) {
        // the GEMMs consume the bf16-rounded gradient: sum exactly what they will read
        uint4 pk = make_uint4(pack_bf16x2(o[0], o[1]), pack_bf16x2(o[2], o[3]), pack_bf16x2(o[4], o[5]), pack_bf16x2(o[6], o[7]));
        const uint32_t* pu = reinterpret_cast<const uint32_t*>(&pk);
        float q[8];
#pragma unroll
        for (int i = 0; i < 4; ++i) { const float2 f = unpack_bf16x2(pu[i]); q[2 * i] = f.x; q[2 * i + 1] = f.y; }
        if (drop_thresh16) {
          const uint64_t lin = (uint64_t)row * (uint64_t)H + (uint64_t)c;
          const uint32_t keep = dropout_keep8(seed, site, lin >> 3, drop_thresh16);
#pragma unroll
          for (int i = 0; i < 8; ++i) q[i] = ((keep >> i) & 1u) ? q[i] * drop_scale : 0.f;
          uint4 mk = make_uint4(pack_bf16x2(q[0], q[1]), pack_bf16x2(q[2], q[3]), pack_bf16x2(q[4], q[5]), pack_bf16x2(q[6], q[7]));
          *reinterpret_cast<uint4*>(dmask + (size_t)row * H + c) = mk;
          const uint32_t* mu2 = reinterpret_cast<const uint32_t*>(&mk);
#pragma unroll
          for (int i = 0; i < 4; ++i) { const float2 f = unpack_bf16x2(mu2[i]); q[2 * i] = f.x; q[2 * i + 1] = f.y; }
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) bs[j][i] += q[i];
      }
    }
    __syncwarp();  // every lane is done reading the slot: refill it with the row LNF_STAGES ahead
    if (k + LNF_STAGES < n_my && leader) {
      fence_proxy_async_smem();
      lnf_issue(ring, bar, k + LNF_STAGES, row + (long long)LNF_STAGES * row_step, x, dy, dres, H);
    }
    if (++stage == LNF_STAGES) { stage = 0; phase ^= 1u; }
  }
  __syncthreads();  // all rings drained (every issued row was waited for): the partials below reuse the ring's bytes
  // warp partials -> smem (plain stores, each warp its own [3][H] slab), summed over the warps by the whole block, then ONE
  // red.global.add per column and block (the same-address reductions of many small blocks used to be the kernel's fixed cost)
  float* mine = sred + (size_t)warp * 3 * H;
#pragma unroll
  for (int j = 0; j < NCH; ++j) {
    const int c = (lane + 32 * j) * 8;
    if (lane + 32 * j >= nchunk) continue;
    *reinterpret_cast<float4*>(mine + c) = make_float4(dg[j][0], dg[j][1], dg[j][2], dg[j][3]);
    *reinterpret_cast<float4*>(mine + c + 4) = make_float4(dg[j][4], dg[j][5], dg[j][6], dg[j][7]);
    *reinterpret_cast<float4*>(mine + H + c) = make_float4(db[j][0], db[j][1], db[j][2], db[j][3]);
    *reinterpret_cast<float4*>(mine + H + c + 4) = make_float4(db[j][4], db[j][5], db[j][6], db[j][7]);
    if (want_bias) {
      *reinterpret_cast<float4*>(mine + 2 * H + c) = make_float4(bs[j][0], bs[j][1], bs[j][2], bs[j][3]);
      *reinterpret_cast<float4*>(mine + 2 * H + c + 4) = make_float4(bs[j][4], bs[j][5], bs[j][6], bs[j][7]);
    }
  }
  __syncthreads();
  for (int i4 = threadIdx.x * 4; i4 < (want_bias ? 3 : 2) * H; i4 += blockDim.x * 4) {  // H % 8 == 0: a float4 never straddles
    float4 a = *reinterpret_cast<const float4*>(sred + i4);
    for (int w = 1; w < nwarp; ++w) {
      const float4 b = *reinterpret_cast<const float4*>(sred + (size_t)w * 3 * H + i4);
      a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
    }
    float* dst = i4 < H ? out_g + i4 : (i4 < 2 * H ? out_b + (i4 - H) : out_bias + (i4 - 2 * H));
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(dst), "f"(a.x), "f"(a.y), "f"(a.z), "f"(a.w) : "memory");
  }
}

// out_k[c] += sum_b partial[b][k*H + c] for k = 0..2 (dgamma, dbeta, bias); grid = (ceil(3H/256), RSPLIT2)
constexpr int RSPLIT2 = 16;
__global__ void reduce_partials3_kernel(const float* __restrict__ partial, int nblocks, int H, float* __restrict__ o0,
                                        float* __restrict__ o1, float* __restrict__ o2) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  const int n = 3 * H;
  if (c >= n) return;
  float* dst = c < H ? o0 + c : (c < 2 * H ? o1 + (c - H) : (o2 ? o2 + (c - 2 * H) : nullptr));
  if (!dst) return;
  float s = 0.f;
  for (int b = blockIdx.y; b < nblocks; b += RSPLIT2) s += partial[(size_t)b * n + c];
  atomicAdd(dst, s);
}

// out[c] += sum_b partial[b][c]   (c in [0, n)); used for LN dgamma/dbeta.  grid = (ceil(n/256), RSPLIT): each thread sums
// every RSPLIT-th partial row, then one fp32 atomic per thread.
constexpr int RSPLIT = 16;
__global__ void reduce_partials_kernel(const float* __restrict__ partial, int nblocks, int n, float* __restrict__ out0,
                                       float* __restrict__ out1, int half) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n) return;
  float s = 0.f;
  for (int b = blockIdx.y; b < nblocks; b += RSPLIT) s += partial[(size_t)b * n + c];
  atomicAdd(c < half ? out0 + c : out1 + (c - half), s);
}

// -----------------------------------------------------------------------------------------------------------------
// bias gradient: out[n] += sum_m dy[m, n]   (optionally through the forward dropout mask)
// grid = (ceil(N/256), row_slabs); block = 256 threads = 8 warps; lane owns 8 columns
// -----------------------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256) colsum_kernel(const T* __restrict__ dy, int ld, long long rows, int N, float* __restrict__ out,
                                                     uint32_t drop_thresh16, float drop_scale, uint64_t seed, uint32_t site) {
  __shared__ float sred[8][256];
  pdl_launch_dependents();
  pdl_wait();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int col = blockIdx.x * 256 + lane * 8;
  float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  if (col < N) {
    for (long long r = (long long)blockIdx.y * 8 + warp; r < rows; r += (long long)gridDim.y * 8) {
      float v[8];
      Vec8<T>::load(dy + (size_t)r * ld + col, v);
      if (drop_thresh16) {
        const uint64_t lin = (uint64_t)r * (uint64_t)N + (uint64_t)col;
        const uint32_t keep = dropout_keep8(seed, site, lin >> 3, drop_thresh16);
#pragma unroll
        for (int i = 0; i < 8; ++i) v[i] = ((keep >> i) & 1u) ? v[i] * drop_scale : 0.f;
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] += v[i];
    }
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) sred[warp][lane * 8 + i] = acc[i];
  __syncthreads();
  const int c = threadIdx.x;
  if (blockIdx.x * 256 + c < N) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) s += sred[w][c];
    atomicAdd(out + blockIdx.x * 256 + c, s);
  }
}

// y = keep ? x * scale : 0  with the forward's (seed, site, row*N+col) indexing
__global__ void dropout_apply_kernel(const bf16* __restrict__ x, int ld_x, bf16* __restrict__ y, int ld_y, long long rows, int N,
                                     uint32_t thresh16, float scale, uint64_t seed, uint32_t site) {
  const long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int per = N >> 3;
  if (gid >= rows * per) return;
  const long long r = gid / per;
  const int c = (int)(gid % per) * 8;
  float v[8];
  Vec8<bf16>::load(x + (size_t)r * ld_x + c, v);
  const uint64_t lin = (uint64_t)r * (uint64_t)N + (uint64_t)c;
  const uint32_t keep = dropout_keep8(seed, site, lin >> 3, thresh16);
#pragma unroll
  for (int i = 0; i < 8; ++i) v[i] = ((keep >> i) & 1u) ? v[i] * scale : 0.f;
  Vec8<bf16>::store(y + (size_t)r * ld_y + c, v);
}

// -----------------------------------------------------------------------------------------------------------------
// row gather: dst[i, :] = src[idx[i], :]   and scatter-add: dst[idx[i], :] += src[i, :]
// -----------------------------------------------------------------------------------------------------------------
template <typename TS, typename TD>
__global__ void gather_rows_kernel(const TS* __restrict__ src, int ld_s, const int* __restrict__ idx, TD* __restrict__ dst, int ld_d,
                                   int n, int H) {
  const long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int per = H >> 3;
  if (gid >= (long long)n * per) return;
  const int i = (int)(gid / per), c = (int)(gid % per) * 8;
  float v[8];
  Vec8<TS>::load(src + (size_t)idx[i] * ld_s + c, v);
  Vec8<TD>::store(dst + (size_t)i * ld_d + c, v);
}
// dst rows may repeat (embedding gradients) -> fp32 atomics; dst is always fp32 here
template <typename TS>
__global__ void scatter_add_rows_kernel(const TS* __restrict__ src, int ld_s, const int* __restrict__ idx, float* __restrict__ dst,
                                        int ld_d, int n, int H, float scale) {
  const long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int per = H >> 3;
  if (gid >= (long long)n * per) return;
  const int i = (int)(gid / per), c = (int)(gid % per) * 8;
  float v[8];
  Vec8<TS>::load(src + (size_t)i * ld_s + c, v);
  float* d = dst + (size_t)idx[i] * ld_d + c;
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(d), "f"(v[0] * scale), "f"(v[1] * scale), "f"(v[2] * scale),
               "f"(v[3] * scale) : "memory");
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(d + 4), "f"(v[4] * scale), "f"(v[5] * scale), "f"(v[6] * scale),
               "f"(v[7] * scale) : "memory");
}
// bf16 destination, unique indices (no collisions): dst[idx[i]] += src[i]
__global__ void scatter_add_rows_bf16_kernel(const float* __restrict__ src, int ld_s, const int* __restrict__ idx, bf16* __restrict__ dst,
                                             int ld_d, int n, int H) {
  const long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int per = H >> 3;
  if (gid >= (long long)n * per) return;
  const int i = (int)(gid / per), c = (int)(gid % per) * 8;
  float v[8], o[8];
  Vec8<float>::load(src + (size_t)i * ld_s + c, v);
  bf16* d = dst + (size_t)idx[i] * ld_d + c;
  Vec8<bf16>::load(d, o);
#pragma unroll
  for (int k = 0; k < 8; ++k) o[k] += v[k];
  Vec8<bf16>::store(d, o);
}

// dx = dy * gelu'(pre)  (fp32, small head tensors)
__global__ void dgelu_kernel(const float* __restrict__ dy, const float* __restrict__ pre, float* __restrict__ dx, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dx[i] = dy[i] * gelu_erf_grad(pre[i]);
}
// y = gelu(x) fp32 -> (fp32, bf16 copy)
__global__ void gelu_kernel(const float* __restrict__ x, float* __restrict__ y, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) y[i] = gelu_erf(x[i]);
}
__global__ void cast_f32_bf16_kernel(const float* __restrict__ x, bf16* __restrict__ y, long long n8) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n8) return;
  float v[8];
  Vec8<float>::load(x + i * 8, v);
  Vec8<bf16>::store(y + i * 8, v);
}
__global__ void cast_bf16_f32_kernel(const bf16* __restrict__ x, float* __restrict__ y, long long n8) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n8) return;
  float v[8];
  Vec8<bf16>::load(x + i * 8, v);
  Vec8<float>::store(y + i * 8, v);
}

// -----------------------------------------------------------------------------------------------------------------
// l2 normalise rows: y = x * rsqrt(max(sum x^2, 1e-12))  (tf.math.l2_normalize);  one warp per row, fp32
// bwd: dx = inv * (dy - y * sum(dy*y))   (clamped rows, sum x^2 < 1e-12: dx = dy * inv)
// The forward stores inv with its sign bit set on clamped rows, so the backward takes the branch the forward took (TF's
// Maximum sends the gradient to sum x^2 when sum x^2 >= eps); no threshold on inv can tell the two apart near 1e-12.
// -----------------------------------------------------------------------------------------------------------------
__global__ void l2norm_fwd_kernel(const float* __restrict__ x, float* __restrict__ y, float* __restrict__ inv_out, int rows, int H) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= rows) return;
  float s = 0.f;
  for (int c = lane; c < H; c += 32) { const float v = x[(size_t)row * H + c]; s += v * v; }
  s = warp_sum(s);
  const bool clamped = s < 1e-12f;
  const float inv = rsqrtf(fmaxf(s, 1e-12f));
  for (int c = lane; c < H; c += 32) y[(size_t)row * H + c] = x[(size_t)row * H + c] * inv;
  if (lane == 0) inv_out[row] = clamped ? -inv : inv;
}
__global__ void l2norm_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ y, const float* __restrict__ inv,
                                  float* __restrict__ dx, int rows, int H) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= rows) return;
  float s = 0.f;
  for (int c = lane; c < H; c += 32) s += dy[(size_t)row * H + c] * y[(size_t)row * H + c];
  s = warp_sum(s);
  const bool clamped = signbit(inv[row]);  // the forward's decision: sum x^2 < 1e-12
  const float iv = fabsf(inv[row]);
  for (int c = lane; c < H; c += 32) {
    const size_t o = (size_t)row * H + c;
    dx[o] = clamped ? dy[o] * iv : iv * (dy[o] - y[o] * s);
  }
}

// -----------------------------------------------------------------------------------------------------------------
// softmax cross-entropy over C classes, one block per row (raw_cross_entropy_with_logits + argmax):
//   fwd: loss[r] = lse - logit[label]; rowmax/rowlse saved; correct[r] = (argmax == label)
//   bwd: dlogits[r, c] = coeff[r] * (softmax - onehot)   (bf16 or fp32 out; padded columns [C, ld) are zeroed)
// -----------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) ce_fwd_kernel(const float* __restrict__ logits, int ld, const int* __restrict__ labels, int C,
                                                     float* __restrict__ loss, float* __restrict__ lse_out, float* __restrict__ correct) {
  __shared__ float sm[8];
  __shared__ int si[8];
  const int r = blockIdx.x;
  const float* row = logits + (size_t)r * ld;
  float mx = -INFINITY;
  int arg = 0x7fffffff;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const float v = row[c];
    if (v > mx) { mx = v; arg = c; }
  }
  // block argmax, first occurrence on ties (tf.argmax)
  for (int o = 16; o > 0; o >>= 1) {
    const float om = __shfl_xor_sync(0xffffffffu, mx, o);
    const int oa = __shfl_xor_sync(0xffffffffu, arg, o);
    if (om > mx || (om == mx && oa < arg)) { mx = om; arg = oa; }
  }
  if ((threadIdx.x & 31) == 0) { sm[threadIdx.x >> 5] = mx; si[threadIdx.x >> 5] = arg; }
  __syncthreads();
  mx = sm[0]; arg = si[0];
  for (int w = 1; w < (blockDim.x >> 5); ++w)
    if (sm[w] > mx || (sm[w] == mx && si[w] < arg)) { mx = sm[w]; arg = si[w]; }
  __syncthreads();
  float s = 0.f;
  for (int c = threadIdx.x; c < C; c += blockDim.x) s += __expf(row[c] - mx);
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int w = 0; w < (blockDim.x >> 5); ++w) t += sm[w];
    const float lse = mx + logf(t);
    const int lab = labels[r];
    loss[r] = lse - row[lab];
    lse_out[r] = lse;
    if (correct) correct[r] = (arg == lab) ? 1.f : 0.f;
  }
}
template <typename TO>
__global__ void __launch_bounds__(256) ce_bwd_kernel(const float* __restrict__ logits, int ld, const int* __restrict__ labels, int C,
                                                     const float* __restrict__ lse, const float* __restrict__ coeff, TO* __restrict__ dlogits,
                                                     int ld_d) {
  const int r = blockIdx.x;
  const float* row = logits + (size_t)r * ld;
  const float l = lse[r], cf = coeff[r];
  const int lab = labels[r];
  for (int c = threadIdx.x; c < ld_d; c += blockDim.x) {
    float g = 0.f;
    if (c < C) g = cf * (__expf(row[c] - l) - (c == lab ? 1.f : 0.f));
    if constexpr (sizeof(TO) == 2) dlogits[(size_t)r * ld_d + c] = __float2bfloat16_rn(g);
    else dlogits[(size_t)r * ld_d + c] = g;
  }
}

static inline uint32_t thresh16(float p) { return (uint32_t)(p * 65536.0f + 0.5f); }

}  // namespace mb

using namespace mb;

// ---- C-ABI ------------------------------------------------------------------------------------------------------
extern "C" int merlot_layernorm_fwd(const merlot_ln_t* d, void* stream_) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
  MB_REQUIRE(d && d->x && d->y && d->gamma && d->beta, MERLOT_EINVAL, "layernorm_fwd: null pointer");
  MB_REQUIRE(d->H % 8 == 0 && d->H <= 1024 && d->H > 0, MERLOT_ESHAPE, "layernorm: H must be a multiple of 8, <= 1024 (got %d)", d->H);
  MB_REQUIRE(d->ld_x % 8 == 0 && d->ld_y % 8 == 0, MERLOT_ESHAPE, "layernorm: leading dims must be multiples of 8");
  if (d->rows == 0) return MERLOT_OK;
  const uint32_t th = d->dropout_p > 0.f ? thresh16(d->dropout_p) : 0;
  const float sc = d->dropout_p > 0.f ? 1.f / (1.f - d->dropout_p) : 1.f;
  const unsigned grid = (unsigned)ceil_div_ll(d->rows, 8);
#define LN_ARGS d->ld_x, (d->y), d->ld_y, d->gamma, d->beta, d->mean, d->rstd, d->rows, d->H, d->eps, d->map_per, d->map_stride, d->map_off, th, sc, d->dropout_seed, d->dropout_site
  if (!d->x_f32 && !d->y_f32)
    MB_CHECK_CUDA(launch_pdl(ln_fwd_kernel<bf16, bf16>, dim3(grid), dim3(256), 0, st, (const bf16*)d->x, d->ld_x, (bf16*)d->y, d->ld_y, d->gamma, d->beta, d->mean, d->rstd, d->rows, d->H, d->eps, d->map_per, d->map_stride, d->map_off, th, sc, d->dropout_seed, d->dropout_site));
  else if (d->x_f32 && !d->y_f32)
    MB_CHECK_CUDA(launch_pdl(ln_fwd_kernel<float, bf16>, dim3(grid), dim3(256), 0, st, (const float*)d->x, d->ld_x, (bf16*)d->y, d->ld_y, d->gamma, d->beta, d->mean, d->rstd, d->rows, d->H, d->eps, d->map_per, d->map_stride, d->map_off, th, sc, d->dropout_seed, d->dropout_site));
  else if (d->x_f32 && d->y_f32)
    MB_CHECK_CUDA(launch_pdl(ln_fwd_kernel<float, float>, dim3(grid), dim3(256), 0, st, (const float*)d->x, d->ld_x, (float*)d->y, d->ld_y, d->gamma, d->beta, d->mean, d->rstd, d->rows, d->H, d->eps, d->map_per, d->map_stride, d->map_off, th, sc, d->dropout_seed, d->dropout_site));
  else
    MB_CHECK_CUDA(launch_pdl(ln_fwd_kernel<bf16, float>, dim3(grid), dim3(256), 0, st, (const bf16*)d->x, d->ld_x, (float*)d->y, d->ld_y, d->gamma, d->beta, d->mean, d->rstd, d->rows, d->H, d->eps, d->map_per, d->map_stride, d->map_off, th, sc, d->dropout_seed, d->dropout_site));
#undef LN_ARGS
  MB_CHECK_LAUNCH();
  return MERLOT_OK;
}

extern "C" size_t merlot_layernorm_bwd_workspace_bytes(int H) { return (size_t)4 * device_sms() * 3 * (size_t)H * sizeof(float); }

extern "C" int merlot_layernorm_bwd(const merlot_ln_bwd_t* d, void* stream_) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
  MB_REQUIRE(d && d->dy && d->x && d->mean && d->rstd && d->gamma && d->dx && d->workspace && d->dgamma && d->dbeta, MERLOT_EINVAL,
             "layernorm_bwd: null pointer");
  MB_REQUIRE(d->H % 8 == 0 && d->H <= 1024 && d->H > 0, MERLOT_ESHAPE, "layernorm_bwd: H must be a multiple of 8, <= 1024");
  if (d->rows == 0) return MERLOT_OK;
  const uint32_t th = d->dropout_p > 0.f ? thresh16(d->dropout_p) : 0;
  const float sc = d->dropout_p > 0.f ? 1.f / (1.f - d->dropout_p) : 1.f;
  long long want = ceil_div_ll(d->rows, 8);
  const int max_grid = 2 * device_sms();  // the workspace holds 2H partials per block for this many blocks (and more)
  const int grid = (int)(want < max_grid ? want : max_grid);
  const size_t smem = (size_t)2 * d->H * sizeof(float);
  float* part = reinterpret_cast<float*>(d->workspace);
#define LNB(TX, TDY, TDX)                                                                                                         \
  ln_bwd_kernel<TX, TDY, TDX><<<grid, 256, smem, st>>>((const TDY*)d->dy, d->ld_dy, (const TX*)d->x, d->ld_x, d->mean, d->rstd,    \
                                                       d->gamma, (const TDX*)d->dres, d->ld_dres, (TDX*)d->dx, d->ld_dx, part,   \
                                                       d->rows, d->H, d->map_per, d->map_stride, d->map_off, th, sc,             \
                                                       d->dropout_seed, d->dropout_site)
  if (!d->x_f32 && !d->dy_f32 && !d->dx_f32) LNB(bf16, bf16, bf16);
  else if (d->x_f32 && !d->dy_f32 && d->dx_f32) LNB(float, bf16, float);
  else if (d->x_f32 && d->dy_f32 && d->dx_f32) LNB(float, float, float);
  else if (!d->x_f32 && d->dy_f32 && !d->dx_f32) LNB(bf16, float, bf16);
  else return set_error(MERLOT_EINVAL, "layernorm_bwd: unsupported dtype combination x_f32=%d dy_f32=%d dx_f32=%d", d->x_f32, d->dy_f32, d->dx_f32);
#undef LNB
  MB_CHECK_LAUNCH();
  reduce_partials_kernel<<<dim3(ceil_div(2 * d->H, 256), RSPLIT), 256, 0, st>>>(part, grid, 2 * d->H, d->dgamma, d->dbeta, d->H);
  MB_CHECK_LAUNCH();
  return MERLOT_OK;
}

extern "C" int merlot_layernorm_bwd_fused(const void* dy, const void* x, const float* mean, const float* rstd, const float* gamma,
                                          const void* dres, void* dx, void* dmask, float* dgamma, float* dbeta, float* dbias,
                                          void* workspace, long long rows, int H, float dropout_p, uint64_t seed, uint32_t site,
                                          void* stream_) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
  MB_REQUIRE(dy && x && mean && rstd && gamma && dx && dgamma && dbeta, MERLOT_EINVAL, "layernorm_bwd_fused: null pointer");
  MB_REQUIRE(H % 8 == 0 && H > 0 && H <= 1024, MERLOT_ESHAPE, "layernorm_bwd_fused: H must be a multiple of 8, <= 1024 (got %d)", H);
  MB_REQUIRE(dropout_p <= 0.f || (dmask && dbias), MERLOT_EINVAL, "layernorm_bwd_fused: dropout needs dmask and dbias");
  if (rows == 0) return MERLOT_OK;
  const uint32_t th = dropout_p > 0.f ? thresh16(dropout_p) : 0;
  const float sc = dropout_p > 0.f ? 1.f / (1.f - dropout_p) : 1.f;
  long long want = ceil_div_ll(rows, LNF_WARPS);
  const int sms = num_sms();
  const int grid = (int)(want < sms ? want : sms);
  const size_t smem = lnf_smem_bytes(H);
  MB_REQUIRE(((reinterpret_cast<uintptr_t>(dy) | reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(dres) |
               reinterpret_cast<uintptr_t>(dx) | reinterpret_cast<uintptr_t>(dmask)) & 15) == 0, MERLOT_EINVAL,
             "layernorm_bwd_fused: dy, x, dres, dx, dmask must be 16-byte aligned");
  (void)workspace;
#define LNF(N_)                                                                                                          \
  do {                                                                                                                   \
    static bool attr_set = false;                                                                                        \
    if (!attr_set) {                                                                                                     \
      MB_CHECK_CUDA(cudaFuncSetAttribute(ln_bwd_fused_kernel<N_>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)lnf_smem_bytes(1024))); \
      attr_set = true;                                                                                                   \
    }                                                                                                                    \
    MB_CHECK_CUDA(launch_pdl(ln_bwd_fused_kernel<N_>, dim3(grid), dim3(32 * LNF_WARPS), smem, st, (const bf16*)dy, (const bf16*)x, mean, \
                             rstd, gamma, (const bf16*)dres, (bf16*)dx, (bf16*)dmask, dgamma, dbeta, dbias, rows, H,     \
                             (int)(dbias != nullptr), th, sc, seed, site));                                              \
  } while (0)
  if (H <= 256) LNF(1); else if (H <= 512) LNF(2); else if (H <= 768) LNF(3); else LNF(4);
#undef LNF
  MB_CHECK_LAUNCH();
  return MERLOT_OK;
}

extern "C" int merlot_bias_grad(const void* dy, int dy_f32, int ld, long long rows, int N, float* out, float dropout_p,
                                uint64_t seed, uint32_t site, void* stream_) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
  MB_REQUIRE(dy && out, MERLOT_EINVAL, "bias_grad: null pointer");
  MB_REQUIRE(N % 8 == 0 && ld % 8 == 0, MERLOT_ESHAPE, "bias_grad: N and ld must be multiples of 8");
  if (rows == 0) return MERLOT_OK;
  const uint32_t th = dropout_p > 0.f ? thresh16(dropout_p) : 0;
  const float sc = dropout_p > 0.f ? 1.f / (1.f - dropout_p) : 1.f;
  long long slabs = ceil_div_ll(rows, 64);
  if (slabs > 128) slabs = 128;
  dim3 grid(ceil_div(N, 256), (unsigned)slabs);
  if (dy_f32) MB_CHECK_CUDA(launch_pdl(colsum_kernel<float>, grid, dim3(256), 0, st, (const float*)dy, ld, rows, N, out, th, sc, seed, site));
  else MB_CHECK_CUDA(launch_pdl(colsum_kernel<bf16>, grid, dim3(256), 0, st, (const bf16*)dy, ld, rows, N, out, th, sc, seed, site));
  MB_CHECK_LAUNCH();
  return MERLOT_OK;
}

extern "C" int merlot_dropout_apply(const void* x, int ld_x, void* y, int ld_y, long long rows, int N, float p, uint64_t seed,
                                    uint32_t site, void* stream_) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
  MB_REQUIRE(x && y, MERLOT_EINVAL, "dropout_apply: null pointer");
  MB_REQUIRE(N % 8 == 0 && p > 0.f && p < 1.f, MERLOT_ESHAPE, "dropout_apply: need N %% 8 == 0 and 0 < p < 1");
  const long long n = rows * (N / 8);
  if (n == 0) return MERLOT_OK;
  dropout_apply_kernel<<<(unsigned)ceil_div_ll(n, 256), 256, 0, st>>>((const bf16*)x, ld_x, (bf16*)y, ld_y, rows, N, thresh16(p),
                                                                       1.f / (1.f - p), seed, site);
  MB_CHECK_LAUNCH();
  return MERLOT_OK;
}

extern "C" int merlot_gather_rows(const void* src, int src_f32, int ld_s, const int* idx, void* dst, int dst_f32, int ld_d, int n,
                                  int H, void* stream_) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
  MB_REQUIRE(src && idx && dst, MERLOT_EINVAL, "gather_rows: null pointer");
  MB_REQUIRE(H % 8 == 0, MERLOT_ESHAPE, "gather_rows: H %% 8 != 0");
  if (n == 0) return MERLOT_OK;
  const unsigned grid = (unsigned)ceil_div_ll((long long)n * (H / 8), 256);
  if (!src_f32 && !dst_f32) gather_rows_kernel<bf16, bf16><<<grid, 256, 0, st>>>((const bf16*)src, ld_s, idx, (bf16*)dst, ld_d, n, H);
  else if (!src_f32 && dst_f32) gather_rows_kernel<bf16, float><<<grid, 256, 0, st>>>((const bf16*)src, ld_s, idx, (float*)dst, ld_d, n, H);
  else if (src_f32 && dst_f32) gather_rows_kernel<float, float><<<grid, 256, 0, st>>>((const float*)src, ld_s, idx, (float*)dst, ld_d, n, H);
  else gather_rows_kernel<float, bf16><<<grid, 256, 0, st>>>((const float*)src, ld_s, idx, (bf16*)dst, ld_d, n, H);
  MB_CHECK_LAUNCH();
  return MERLOT_OK;
}

extern "C" int merlot_scatter_add_rows(const void* src, int src_f32, int ld_s, const int* idx, void* dst, int dst_f32, int ld_d,
                                       int n, int H, float scale, void* stream_) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
  MB_REQUIRE(src && idx && dst, MERLOT_EINVAL, "scatter_add_rows: null pointer");
  MB_REQUIRE(H % 8 == 0, MERLOT_ESHAPE, "scatter_add_rows: H %% 8 != 0");
  if (n == 0) return MERLOT_OK;
  const unsigned grid = (unsigned)ceil_div_ll((long long)n * (H / 8), 256);
  if (dst_f32) {
    if (src_f32) scatter_add_rows_kernel<float><<<grid, 256, 0, st>>>((const float*)src, ld_s, idx, (float*)dst, ld_d, n, H, scale);
    else scatter_add_rows_kernel<bf16><<<grid, 256, 0, st>>>((const bf16*)src, ld_s, idx, (float*)dst, ld_d, n, H, scale);
  } else {
    MB_REQUIRE(src_f32 && scale == 1.0f, MERLOT_EINVAL, "scatter_add_rows: bf16 destination needs fp32 source, scale 1, unique idx");
    scatter_add_rows_bf16_kernel<<<grid, 256, 0, st>>>((const float*)src, ld_s, idx, (bf16*)dst, ld_d, n, H);
  }
  MB_CHECK_LAUNCH();
  return MERLOT_OK;
}

extern "C" int merlot_gelu_f32(const float* x, float* y, long long n, void* stream_) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
  MB_REQUIRE(x && y, MERLOT_EINVAL, "gelu_f32: null pointer");
  if (n == 0) return MERLOT_OK;
  gelu_kernel<<<(unsigned)ceil_div_ll(n, 256), 256, 0, st>>>(x, y, n);
  MB_CHECK_LAUNCH();
  return MERLOT_OK;
}
extern "C" int merlot_gelu_bwd_f32(const float* dy, const float* pre, float* dx, long long n, void* stream_) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
  MB_REQUIRE(dy && pre && dx, MERLOT_EINVAL, "gelu_bwd_f32: null pointer");
  if (n == 0) return MERLOT_OK;
  dgelu_kernel<<<(unsigned)ceil_div_ll(n, 256), 256, 0, st>>>(dy, pre, dx, n);
  MB_CHECK_LAUNCH();
  return MERLOT_OK;
}
extern "C" int merlot_cast_f32_to_bf16(const float* x, void* y, long long n, void* stream_) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
  MB_REQUIRE(x && y, MERLOT_EINVAL, "cast: null pointer");
  MB_REQUIRE(n % 8 == 0, MERLOT_ESHAPE, "cast: n %% 8 != 0");
  if (n == 0) return MERLOT_OK;
  cast_f32_bf16_kernel<<<(unsigned)ceil_div_ll(n / 8, 256), 256, 0, st>>>(x, (bf16*)y, n / 8);
  MB_CHECK_LAUNCH();
  return MERLOT_OK;
}
extern "C" int merlot_cast_bf16_to_f32(const void* x, float* y, long long n, void* stream_) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
  MB_REQUIRE(x && y, MERLOT_EINVAL, "cast: null pointer");
  MB_REQUIRE(n % 8 == 0, MERLOT_ESHAPE, "cast: n %% 8 != 0");
  if (n == 0) return MERLOT_OK;
  cast_bf16_f32_kernel<<<(unsigned)ceil_div_ll(n / 8, 256), 256, 0, st>>>((const bf16*)x, y, n / 8);
  MB_CHECK_LAUNCH();
  return MERLOT_OK;
}

extern "C" int merlot_l2norm_fwd(const float* x, float* y, float* inv, int rows, int H, void* stream_) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
  MB_REQUIRE(x && y && inv, MERLOT_EINVAL, "l2norm_fwd: null pointer");
  if (rows == 0) return MERLOT_OK;
  l2norm_fwd_kernel<<<ceil_div(rows, 8), 256, 0, st>>>(x, y, inv, rows, H);
  MB_CHECK_LAUNCH();
  return MERLOT_OK;
}
extern "C" int merlot_l2norm_bwd(const float* dy, const float* y, const float* inv, float* dx, int rows, int H, void* stream_) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
  MB_REQUIRE(dy && y && inv && dx, MERLOT_EINVAL, "l2norm_bwd: null pointer");
  if (rows == 0) return MERLOT_OK;
  l2norm_bwd_kernel<<<ceil_div(rows, 8), 256, 0, st>>>(dy, y, inv, dx, rows, H);
  MB_CHECK_LAUNCH();
  return MERLOT_OK;
}

extern "C" int merlot_softmax_ce_fwd(const float* logits, int ld, const int* labels, int rows, int C, float* loss, float* lse,
                                     float* correct, void* stream_) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
  MB_REQUIRE(logits && labels && loss && lse, MERLOT_EINVAL, "softmax_ce_fwd: null pointer");
  MB_REQUIRE(C > 0 && ld >= C, MERLOT_ESHAPE, "softmax_ce_fwd: need 0 < C <= ld");
  if (rows == 0) return MERLOT_OK;
  ce_fwd_kernel<<<rows, 256, 0, st>>>(logits, ld, labels, C, loss, lse, correct);
  MB_CHECK_LAUNCH();
  return MERLOT_OK;
}
extern "C" int merlot_softmax_ce_bwd(const float* logits, int ld, const int* labels, int rows, int C, const float* lse,
                                     const float* coeff, void* dlogits, int dlogits_f32, int ld_d, void* stream_) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
  MB_REQUIRE(logits && labels && lse && coeff && dlogits, MERLOT_EINVAL, "softmax_ce_bwd: null pointer");
  MB_REQUIRE(C > 0 && ld >= C && ld_d >= C, MERLOT_ESHAPE, "softmax_ce_bwd: need 0 < C <= ld, ld_d");
  if (rows == 0) return MERLOT_OK;
  if (dlogits_f32) ce_bwd_kernel<float><<<rows, 256, 0, st>>>(logits, ld, labels, C, lse, coeff, (float*)dlogits, ld_d);
  else ce_bwd_kernel<bf16><<<rows, 256, 0, st>>>(logits, ld, labels, C, lse, coeff, (bf16*)dlogits, ld_d);
  MB_CHECK_LAUNCH();
  return MERLOT_OK;
}
