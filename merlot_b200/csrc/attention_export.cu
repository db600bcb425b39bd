// Head-mean attention probabilities of one layer, materialised: `self_attn_probs` of utils/transformer.py:208-209,238
// (compress_attn=True: tf.reduce_mean(attn_probs, 1)), which model_fn's PREDICT mode returns (model/modeling.py:762-770).
// An export path, not a hot one: the probabilities are recomputed from the saved (q, k, log-sum-exp) with plain fp32 dot
// products -- [B, S, S] fp32 per layer would be 60 MB per joint layer at configs[1], which is why the training path never
// materialises them (K2/K3/K4 keep them on chip).
#include "host_common.h"
#include "ptx.cuh"

namespace mb {

constexpr int EXQ = 8;  // query rows per CTA

// keep bit of probability (q, k) of head h under attention-probability dropout, one element at a time (ptx.cuh
// attn_dropout_words; K2/K3/K4 draw the same bits four per call)
__device__ __forceinline__ bool attn_keep_one(uint64_t seed, uint32_t site, uint32_t thresh16, int b, int heads, int h, int S, int q, int k) {
  const uint64_t n16 = (uint64_t)((S + 15) >> 4);
  const uint64_t blk = (((((uint64_t)b * heads + h) * n16 + (uint64_t)(q >> 4)) * 8 + (q & 7)) * n16 + (uint64_t)(k >> 4)) * 8 + (k & 7);
  const uint4 r = attn_dropout_words(seed, site, blk);
  const uint32_t w = ((q >> 3) & 1) ? (((k >> 3) & 1) ? r.w : r.z) : (((k >> 3) & 1) ? r.y : r.x);
  return (w >> 16) >= thresh16;
}

// grid (ceil(S / EXQ), B); 256 threads, thread t walks keys t, t + 256, ...
// DROP: the head mean of the dropped probabilities P o Z / (1 - p) (self_attn_probs is built from them, transformer.py:138)
template <bool DROP>
__global__ void __launch_bounds__(256) attn_probs_export_kernel(const bf16* __restrict__ qkv, int ld_qkv, const uint8_t* __restrict__ valid,
                                                                const float* __restrict__ lse, float* __restrict__ out, int B, int S,
                                                                int heads, float scale, int pair_P, int pair_chunk, uint32_t drop_thresh16,
                                                                float drop_scale, uint64_t drop_seed, uint32_t drop_site) {
  extern __shared__ float sm[];
  const int H = heads * 64;
  float* sq = sm;                 // [EXQ][H]   queries of this CTA (fp32), pre-scaled
  float* sl = sm + EXQ * H;       // [EXQ][heads] log-sum-exp
  const int b = blockIdx.y, q0 = blockIdx.x * EXQ, tok0 = b * S;
  for (int i = threadIdx.x; i < EXQ * H; i += 256) {
    const int r = i / H, c = i % H, q = q0 + r;
    sq[i] = (q < S) ? __bfloat162float(qkv[(size_t)(tok0 + q) * ld_qkv + c]) * scale : 0.f;
  }
  for (int i = threadIdx.x; i < EXQ * heads; i += 256) {
    const int r = i / heads, hh = i % heads, q = q0 + r;
    sl[i] = (q < S) ? lse[((size_t)b * heads + hh) * S + q] : 0.f;
  }
  __syncthreads();
  bool vq[EXQ];
#pragma unroll
  for (int r = 0; r < EXQ; ++r) vq[r] = (q0 + r < S) && (valid == nullptr || valid[tok0 + q0 + r] != 0);
  // disable_pairwise_lang_attn (model/modeling.py:160-168): segment of a position = 0 for the pair_P vision tokens, 1 + chunk index
  // otherwise; a pair attends iff same segment or either is a vision token
  auto seg_of = [&](int t) { return (pair_chunk > 0 && t >= pair_P) ? 1 + (t - pair_P) / pair_chunk : 0; };
  int sq_seg[EXQ];
#pragma unroll
  for (int r = 0; r < EXQ; ++r) sq_seg[r] = seg_of(q0 + r);
  const float inv_heads = (DROP ? drop_scale : 1.0f) / (float)heads;
  for (int k = threadIdx.x; k < S; k += 256) {
    const bool vk = valid == nullptr || valid[tok0 + k] != 0;
    const int k_seg = seg_of(k);
    float acc[EXQ];
#pragma unroll
    for (int r = 0; r < EXQ; ++r) acc[r] = 0.f;
    const bf16* krow = qkv + (size_t)(tok0 + k) * ld_qkv + H;
    for (int hh = 0; hh < heads; ++hh) {
      float dot[EXQ];
#pragma unroll
      for (int r = 0; r < EXQ; ++r) dot[r] = 0.f;
#pragma unroll
      for (int c8 = 0; c8 < 8; ++c8) {
        const uint4 u = __ldg(reinterpret_cast<const uint4*>(krow + hh * 64 + c8 * 8));
        const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 f = unpack_bf16x2(w[j]);
          const int c = hh * 64 + c8 * 8 + j * 2;
#pragma unroll
          for (int r = 0; r < EXQ; ++r) dot[r] = fmaf(sq[r * H + c], f.x, fmaf(sq[r * H + c + 1], f.y, dot[r]));
        }
      }
#pragma unroll
      for (int r = 0; r < EXQ; ++r) {
        // utils/transformer.py:109-112: scores*m - 1e10*(1-m); a padding query row has every score equal => uniform
        const bool pair_ok = k_seg == 0 || sq_seg[r] == 0 || k_seg == sq_seg[r];
        const float s = !vq[r] ? 0.f : ((vk && pair_ok) ? dot[r] : -1e10f);
        const float pr = __expf(s - sl[r * heads + hh]);
        if (DROP) acc[r] += attn_keep_one(drop_seed, drop_site, drop_thresh16, b, heads, hh, S, q0 + r, k) ? pr : 0.f;
        else acc[r] += pr;
      }
    }
#pragma unroll
    for (int r = 0; r < EXQ; ++r)
      if (q0 + r < S) out[((size_t)b * S + q0 + r) * S + k] = acc[r] * inv_heads;
  }
}

}  // namespace mb

using namespace mb;

extern "C" int merlot_attention_probs(const merlot_attn_t* a, float* probs_bss, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  MB_REQUIRE(a && probs_bss && a->qkv && a->lse, MERLOT_EINVAL, "attention_probs: qkv, lse and the output are required");
  MB_REQUIRE(a->head_dim == 64 && a->B > 0 && a->S > 0 && a->heads > 0 && (a->ld_qkv % 8) == 0, MERLOT_ESHAPE,
             "attention_probs: head size 64, ld_qkv %% 8 == 0");
  MB_REQUIRE(a->pair_chunk_len >= 0 && a->pair_viz_len >= 0 && (a->pair_chunk_len == 0 || a->valid != nullptr), MERLOT_EINVAL,
             "attention_probs: pair_chunk_len > 0 (disable_pairwise_lang_attn) needs the token-validity mask");
  MB_REQUIRE(a->dropout_p >= 0.f && a->dropout_p < 1.f, MERLOT_EINVAL, "attention_probs: dropout_p must lie in [0, 1) (got %g)",
             (double)a->dropout_p);
  const int H = a->heads * 64;
  const size_t smem = (size_t)(EXQ * H + EXQ * a->heads) * sizeof(float);
  MB_REQUIRE(smem <= 200 * 1024, MERLOT_ESHAPE, "attention_probs: hidden size too large");
  static size_t attr = 0;
  if (smem > attr) {
    MB_CHECK_CUDA(cudaFuncSetAttribute(attn_probs_export_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    MB_CHECK_CUDA(cudaFuncSetAttribute(attn_probs_export_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr = smem;
  }
  dim3 grid(ceil_div(a->S, EXQ), a->B);
  // the same float32 quantisation as K2/K3/K4 (attention.cu fill_dev)
  const uint32_t th = (uint32_t)(a->dropout_p * 65536.0f + 0.5f);
  const float ds = 1.0f / (1.0f - a->dropout_p);
  auto kern = a->dropout_p > 0.f ? attn_probs_export_kernel<true> : attn_probs_export_kernel<false>;
  kern<<<grid, 256, smem, stream>>>(reinterpret_cast<const bf16*>(a->qkv), a->ld_qkv, reinterpret_cast<const uint8_t*>(a->valid), a->lse,
                                    probs_bss, a->B, a->S, a->heads, a->scale, a->pair_viz_len, a->pair_chunk_len, th, ds,
                                    a->dropout_seed, a->dropout_site);
  MB_CHECK_LAUNCH();
  return MERLOT_OK;
}
