// K2/K3/K4: masked softmax attention on wgmma tensor cores, FlashAttention-style (probabilities never hit HBM).
//
// Replaces utils/transformer.py:98-127 (scores = q k^T / sqrt(d); scores*m - 1e10*(1-m); softmax; probs @ v) and its
// tf.gradients, plus the consumers of the materialised probabilities: the head-mean column sums that
// model/modeling.py:428 (mask_inputs) takes from `self_attn_probs` (utils/transformer.py:208-209,238).
//
// Layout: q/k/v are read in place from the fused QKV GEMM output [tokens, 3H] (columns [0,H) = q, [H,2H) = k,
// [2H,3H) = v, head h at column h*64) through 2-D TMA maps; ctx / d_ctx are [tokens, H].  Head size is 64.
//
// Mask semantics (reference :109-112, SURVEY quirk 8): m[q,k] = valid[q] & valid[k].  A masked entry's score is
// exactly -1e10; a padding QUERY row therefore has all scores equal and softmaxes to uniform 1/S over all S keys.
// We realise that row as all-zero scores (identical softmax, but keeps log-sum-exp = log S representable).
//
// Every kernel runs two warpgroups of 128 threads; each owns 64 rows of the tile (one m64 wgmma).  Accumulator element
// d[4j + 2i + e] of a thread is row (16 w + l/4 + 8 i) and column (8 j + 2 (l%4) + e) of its warpgroup's block (ptx.cuh).
#include "host_common.h"
#include "ptx.cuh"

namespace mb {

constexpr int AT_M = 128;   // query rows per forward tile
constexpr int AT_N = 128;   // keys per backward / column-sum tile
constexpr int AT_D = 64;    // head size
constexpr float LOG2E = 1.4426950408889634f;
constexpr float LN2 = 0.6931471805599453f;

struct AttnDev {
  int B, S, heads, H;
  const uint8_t* valid;  // [B*S] or null (all valid)
  float scale;
  bf16* ctx; int ld_ctx;         // fwd out [B*S, H]
  float* lse;                    // [B, heads, S] natural-log LSE of the masked, scaled scores
  // backward
  float* dsum;                   // [B, heads, S]  D = rowsum(dO * O)
  float* dq_accum; int ld_dq;    // fp32 [B*S, H], atomically accumulated by K3 (sequences of more than 512 tokens)
  bf16* dqkv; int ld_dqkv;       // bf16 [B*S, 3H]
  float* d_bias;                 // optional [3H] += column sums of dqkv (the short-sequence kernels add them in their epilogues)
  // K4
  float* colsum;                 // [B, S] += sum_q mean_h P[b,h,q,k]
  float* colsum2;                // optional: queries >= colsum_split accumulate here instead
  int colsum_split;              // 0 = no split
  int colsum_valid_q;            // 1 = only valid (non-padding) queries contribute (attention_log, modeling.py:192-193)
  int pair_P, pair_chunk;        // disable_pairwise_lang_attn (model/modeling.py:160-168); pair_chunk == 0: off
  // attention-probability dropout (DROP instances only; utils/transformer.py:114-115): keep <=> lane16 >= drop_thresh16
  uint32_t drop_thresh16;
  float drop_scale;              // 1 / (1 - p)
  uint64_t drop_seed;
  uint32_t drop_site;
};

constexpr int MAX_MASK_WORDS = 128;  // validity bitmask for up to 4096 positions
constexpr float MASKED_LOG2 = -1e10f * LOG2E;

// bitmask of in-range positions for the 32-position word starting at k
__device__ __forceinline__ uint32_t range_word(int k, int S) {
  const int n = S - k;
  return n >= 32 ? 0xffffffffu : (n <= 0 ? 0u : ((1u << n) - 1u));
}

// bits of the 32-position word starting at x0 whose positions lie in [a, b)
__device__ __forceinline__ uint32_t span_word(int x0, int a, int b) {
  const int lo = max(a - x0, 0), hi = min(b - x0, 32);
  if (hi <= lo) return 0u;
  const uint32_t below_hi = hi >= 32 ? 0xffffffffu : ((1u << hi) - 1u);
  return below_hi & (0xffffffffu << lo);
}
// disable_pairwise_lang_attn (model/modeling.py:160-168): segment 0 = the P vision tokens, segment 1 + c = language chunk c;
// two positions exchange attention iff they share a segment or either is a vision token.  The relation is symmetric, so one
// helper serves "keys a query may see" (K2) and "queries a key is seen by" (K3, K4).  pair_lo_of: start of the language chunk
// of position t, or -1 when t is unrestricted (vision token / feature off); pair_word: the partners of such a position
// inside the 32-position word starting at x0.
__device__ __forceinline__ int pair_lo_of(int t, int P, int chunk) {
  return (chunk > 0 && t >= P) ? P + ((t - P) / chunk) * chunk : -1;
}
__device__ __forceinline__ uint32_t pair_word(int x0, int lo, int P, int chunk) {
  return lo < 0 ? 0xffffffffu : (span_word(x0, 0, P) | span_word(x0, lo, lo + chunk));
}

// validity bits of positions [0, n) of one batch element into s_mask (bit k%32 of word k/32); all threads of the block
__device__ __forceinline__ void build_mask(uint32_t* s_mask, const uint8_t* valid, int n, int S) {
  for (int k = threadIdx.x; k < n; k += blockDim.x) {
    const bool v = (k < S) ? (valid[k] != 0) : false;
    const uint32_t w = __ballot_sync(0xffffffffu, v);
    if ((threadIdx.x & 31) == 0) s_mask[k >> 5] = w;
  }
}

// the A fragment of k-step kk (columns [16 kk, 16 kk + 16)) from an m64n64 accumulator, rounded to bf16
__device__ __forceinline__ void acc_to_afrag(const float (&d)[32], int kk, uint32_t (&a)[4]) {
  a[0] = pack_bf16x2(d[8 * kk + 0], d[8 * kk + 1]);
  a[1] = pack_bf16x2(d[8 * kk + 2], d[8 * kk + 3]);
  a[2] = pack_bf16x2(d[8 * kk + 4], d[8 * kk + 5]);
  a[3] = pack_bf16x2(d[8 * kk + 6], d[8 * kk + 7]);
}

__device__ __forceinline__ void quad_max(float& x) {
  x = fmaxf(x, __shfl_xor_sync(0xffffffffu, x, 1));
  x = fmaxf(x, __shfl_xor_sync(0xffffffffu, x, 2));
}
__device__ __forceinline__ void quad_sum(float& x) {
  x += __shfl_xor_sync(0xffffffffu, x, 1);
  x += __shfl_xor_sync(0xffffffffu, x, 2);
}

// Attention-probability dropout with queries on the accumulator rows (K2, the dQ kernel): bit 4 jj + 2 i + e of the result is
// the keep bit of accumulator element s[4 jj + 2 i + e] of this thread in the 64-key tile starting at k0 (ptx.cuh
// attn_dropout_words: word 2 (q/8 & 1) + (k/8 & 1), with q/8 & 1 = i and k/8 & 1 = jj & 1 here).  drop_row = the query terms.
__device__ __forceinline__ uint32_t attn_keep_bits_queryrows(const AttnDev& p, uint64_t drop_row, int k0, int lane) {
  uint32_t z = 0;
#pragma unroll
  for (int jp = 0; jp < 4; ++jp) {
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const uint4 r = attn_dropout_words(p.drop_seed, p.drop_site, drop_row + (uint64_t)((k0 >> 4) + jp) * 8 + 2 * (lane & 3) + e);
      const uint32_t w[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
      for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int kh = 0; kh < 2; ++kh)  // accumulator column group jj = 2 jp + kh
          z |= ((w[2 * i + kh] >> 16) >= p.drop_thresh16 ? 1u : 0u) << (4 * (2 * jp + kh) + 2 * i + e);
    }
  }
  return z;
}

// Adds the column sums of a warpgroup's 64 x 64 bf16 output block (this thread's values v[4 jj + 2 i + e], already rounded to
// bf16 and zero in rows that are not written) to bias[8 jj + 2 (lane % 4) + e]: a sum over the 8 row groups of the warp by
// shuffles, over the 4 warps through s_red [4][64], then one atomicAdd per column.  Every thread of the (one-warpgroup) CTA
// calls it.
__device__ __forceinline__ void bias_colsum_add(float (&v)[32], float* s_red, float* bias, int wq, int lane, int tid) {
  float c[16];
#pragma unroll
  for (int jj = 0; jj < 8; ++jj)
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      float x = v[4 * jj + e] + v[4 * jj + 2 + e];
      x += __shfl_xor_sync(0xffffffffu, x, 4);
      x += __shfl_xor_sync(0xffffffffu, x, 8);
      x += __shfl_xor_sync(0xffffffffu, x, 16);
      c[2 * jj + e] = x;
    }
  if (lane < 4) {
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) {
      s_red[wq * 64 + 8 * jj + 2 * lane] = c[2 * jj];
      s_red[wq * 64 + 8 * jj + 2 * lane + 1] = c[2 * jj + 1];
    }
  }
  __syncthreads();
  if (tid < 64) atomicAdd(bias + tid, ((s_red[tid] + s_red[64 + tid]) + s_red[128 + tid]) + s_red[192 + tid]);
}

// -----------------------------------------------------------------------------------------------------------------
// forward.  One CTA per (128-query tile, head, batch); warpgroup w owns queries [64 w, 64 w + 64).  Key tiles of 64 run
// through a two-buffer TMA ring.  Per key tile:  S = Q K^T (wgmma, smem x smem) -> masked online softmax in registers (key
// validity as register bitmasks) -> P (bf16) straight from the S accumulator into the A registers of O += P V (wgmma,
// registers x smem), O accumulated in registers.
// -----------------------------------------------------------------------------------------------------------------
constexpr int FK = 64;  // keys per tile
constexpr int FWD_THREADS = 256;
constexpr int FWD_SMEM = 16384 + 2 * 16384 + 512 + 64 + 1024;  // Q, 2 x {K, V}, masks, barriers, alignment

template <bool HAS_MASK, bool DROP>
__global__ void __launch_bounds__(FWD_THREADS, 2) attn_fwd_kernel(const __grid_constant__ CUtensorMap tm_q, const __grid_constant__ CUtensorMap tm_kv,
                                                                  const AttnDev p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;
  uint8_t* sKV = smem + 16384;  // [2] x { K tile 8 KB, V tile 8 KB }: tile j lives in buffer j & 1
  uint32_t* s_mask = reinterpret_cast<uint32_t*>(smem + 49152);  // [MAX_MASK_WORDS]
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + 49152 + 512);
  uint64_t *bar_q = bars, *bar_kv = bars + 1 /* [2] */;

  const int tid = threadIdx.x, lane = tid & 31;
  const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);
  const int wg = warp >> 2, wq = warp & 3;
  const int q0 = blockIdx.x * AT_M, h = blockIdx.y, b = blockIdx.z;
  pdl_launch_dependents();
  const int S = p.S, H = p.H;
  const int tok0 = b * S;
  const int n_kv = (S + FK - 1) / FK;
  static_assert(FK == 64, "attn_keep_bits_queryrows draws the bits of 64-key tiles");

  if (tid == 0) {
    tma_prefetch_desc(&tm_q); tma_prefetch_desc(&tm_kv);
    mbar_init(bar_q, 1); mbar_init(&bar_kv[0], 1); mbar_init(&bar_kv[1], 1);
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();
  auto load_kv = [&](int j) {
    uint8_t* buf = sKV + (j & 1) * 16384;
    mbar_arrive_expect_tx(&bar_kv[j & 1], 16384);
    tma_load_2d(buf, &tm_kv, &bar_kv[j & 1], H + h * AT_D, tok0 + j * FK);
    tma_load_2d(buf + 8192, &tm_kv, &bar_kv[j & 1], 2 * H + h * AT_D, tok0 + j * FK);
  };
  if (tid == 0) {
    mbar_arrive_expect_tx(bar_q, 16384);
    tma_load_2d(sQ, &tm_q, bar_q, h * AT_D, tok0 + q0);
    load_kv(0);
    if (n_kv > 1) load_kv(1);
  }
  if (HAS_MASK) build_mask(s_mask, p.valid + tok0, n_kv * FK, S);
  __syncthreads();

  // this thread's two query rows (i = 0, 1)
  bool q_in[2];
  float sc2[2], m_run[2], l_run[2];
  int pair_lo[2];
  bool vq[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int q = q0 + wg * 64 + wq * 16 + (lane >> 2) + 8 * i;
    q_in[i] = q < S;
    vq[i] = (HAS_MASK && q_in[i]) ? (p.valid[tok0 + q] != 0) : true;
    // a padding QUERY row softmaxes uniformly over all in-range keys: realised as zero scores with every key "valid"
    sc2[i] = vq[i] ? p.scale * LOG2E : 0.f;
    pair_lo[i] = (HAS_MASK && vq[i]) ? pair_lo_of(q, p.pair_P, p.pair_chunk) : -1;
    m_run[i] = -INFINITY;
    l_run[i] = 0.f;
  }
  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  // dropout block index of this thread's queries {q, q + 8} (ptx.cuh attn_dropout_words) up to the key terms
  uint64_t drop_row = 0;
  if (DROP) {
    const uint64_t n16 = (uint64_t)((S + 15) >> 4);
    drop_row = ((((uint64_t)b * p.heads + h) * n16 + (uint64_t)((q0 + wg * 64 + wq * 16) >> 4)) * 8 + (lane >> 2)) * n16 * 8;
  }

  mbar_wait(bar_q, 0);
  const uint32_t qa = smem_u32(sQ) + wg * 8192;
  for (int j = 0; j < n_kv; ++j) {
    // keep bits of this key tile, drawn while only O is live: with S live as well the no-mask instance would spill at 128
    // registers
    const uint32_t zq = DROP ? attn_keep_bits_queryrows(p, drop_row, j * FK, lane) : 0u;
    mbar_wait(&bar_kv[j & 1], (uint32_t)((j >> 1) & 1));
    const uint32_t ka = smem_u32(sKV + (j & 1) * 16384), va = ka + 8192;
    float s[32];
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < AT_D / 16; ++k) wgmma_m64n64_ss<0, 0>(s, desc_kmajor(qa, k), desc_kmajor(ka, k), k > 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(s);
    const int k0 = j * FK;
    // ---- masked scores (log2 domain), online softmax ----
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      uint32_t iw[2], vw[2];
#pragma unroll
      for (int w = 0; w < 2; ++w) {
        iw[w] = range_word(k0 + 32 * w, S);
        vw[w] = (HAS_MASK && vq[i]) ? s_mask[(k0 >> 5) + w] : 0xffffffffu;
        if (HAS_MASK && pair_lo[i] >= 0) vw[w] &= pair_word(k0 + 32 * w, pair_lo[i], p.pair_P, p.pair_chunk);
      }
      float mx = -INFINITY;
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int bit = (8 * jj + 2 * (lane & 3) + e) & 31, w = jj >> 2;
          float t = s[4 * jj + 2 * i + e] * sc2[i];
          t = ((vw[w] >> bit) & 1u) ? t : MASKED_LOG2;
          t = ((iw[w] >> bit) & 1u) ? t : -INFINITY;
          s[4 * jj + 2 * i + e] = t;
          mx = fmaxf(mx, t);
        }
      }
      quad_max(mx);
      const float m_new = fmaxf(m_run[i], mx);
      const float f = ex2_approx(m_run[i] - m_new);  // 0 on the first tile (m_run = -inf)
      m_run[i] = m_new;
      float rs = 0.f;
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float pr = ex2_approx(s[4 * jj + 2 * i + e] - m_new);
          s[4 * jj + 2 * i + e] = pr;
          rs += pr;
          o[4 * jj + 2 * i + e] *= f;
        }
      }
      l_run[i] = l_run[i] * f + rs;
    }
    if (DROP) {  // P o Z after l_run took the undropped sum; the 1/(1-p) rides on the final 1/l
#pragma unroll
      for (int x = 0; x < 32; ++x)
        if (!((zq >> x) & 1u)) s[x] = 0.f;
    }
    // ---- O += P V (P from registers, V MN-major: rows are keys) ----
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < FK / 16; ++kk) {
      uint32_t a[4];
      acc_to_afrag(s, kk, a);
      wgmma_m64n64_rs<1>(o, a, desc_mnmajor(va, kk, 0), 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(o);
    __syncthreads();  // both warpgroups are done with buffer j & 1
    if (tid == 0 && j + 2 < n_kv) load_kv(j + 2);
  }

#pragma unroll
  for (int i = 0; i < 2; ++i) {
    quad_sum(l_run[i]);
    const int q = q0 + wg * 64 + wq * 16 + (lane >> 2) + 8 * i;
    if (!q_in[i]) continue;
    const float inv = (DROP ? p.drop_scale : 1.0f) / l_run[i];
    bf16* dst = p.ctx + (size_t)(tok0 + q) * p.ld_ctx + h * AT_D + 2 * (lane & 3);
#pragma unroll
    for (int jj = 0; jj < 8; ++jj)
      *reinterpret_cast<uint32_t*>(dst + 8 * jj) = pack_bf16x2(o[4 * jj + 2 * i] * inv, o[4 * jj + 2 * i + 1] * inv);
    if ((lane & 3) == 0 && p.lse) p.lse[((size_t)b * p.heads + h) * S + q] = (m_run[i] + log2f(l_run[i])) * LN2;
  }
}

// -----------------------------------------------------------------------------------------------------------------
// backward.  One CTA per (128-key tile, head, batch); warpgroup w owns keys [64 w, 64 w + 64).  The queries are walked in
// chunks of 64 through a two-buffer TMA ring (Q and dO chunk, plus the chunk's -lse*log2(e) and D staged in smem).  Per chunk:
//   S^T = K Q^T, dP^T = V dO^T                       (wgmma, smem x smem, registers)
//   P^T = exp2(S^T sc - lse), dS'^T = P^T (dP^T - D)  (registers)
//   dV += P^T dO, dK += dS'^T Q                        (wgmma, A = P^T / dS'^T straight from registers)
//   dS'^T -> bf16 smem; dQ_chunk = dS' K               (wgmma, both operands MN-major; warpgroup w computes head columns
//                                                       [32 w, 32 w + 32) over all 128 keys) -> fp32 stores of the partial
// 1/sqrt(d) is applied once per output (dK in the epilogue, dQ in attn_dqkv_finish) instead of once per score.
// dQ is red.add-ed into one fp32 slice of the workspace.  K3 serves sequences of more than MAX_DQ_PARTS key tiles; shorter
// ones take the two short-sequence kernels below.
// -----------------------------------------------------------------------------------------------------------------
constexpr int BQ = 64;              // queries per chunk
constexpr int MAX_DQ_PARTS = 4;     // key tiles of 128 up to which the short-sequence kernels run (S <= 512)
constexpr int BWD_THREADS = 256;
// K, V (16 KB each), 2 x {Q, dO} chunk (8 KB each), dS^T 16 KB, statistics 2 x 2 x 256 B, query mask, barriers, alignment
constexpr int BWD_SMEM = 32768 + 32768 + 16384 + 1024 + 512 + 64 + 1024;

// Attention-probability dropout with keys on the accumulator rows (K3, K4): bit 4 jj + 2 i + e of the result is the keep bit of
// accumulator element s[4 jj + 2 i + e] of this thread in the query chunk starting at q0 (ptx.cuh attn_dropout_words: word
// 2 (q/8 & 1) + (k/8 & 1), with q/8 & 1 = jj & 1 and k/8 & 1 = i here).  drop_bh = (b heads + h) n16; drop_key = the key terms.
__device__ __forceinline__ uint32_t attn_keep_bits_keyrows(const AttnDev& p, uint64_t drop_bh, uint64_t drop_key, uint64_t n16, int q0,
                                                           int lane) {
  uint32_t z = 0;
#pragma unroll
  for (int jp = 0; jp < BQ / 16; ++jp) {
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const uint64_t blk = ((drop_bh + (uint64_t)((q0 >> 4) + jp)) * 8 + 2 * (lane & 3) + e) * n16 * 8 + drop_key;
      const uint4 r = attn_dropout_words(p.drop_seed, p.drop_site, blk);
      const uint32_t w[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
      for (int qh = 0; qh < 2; ++qh)
#pragma unroll
        for (int i = 0; i < 2; ++i)
          z |= ((w[2 * qh + i] >> 16) >= p.drop_thresh16 ? 1u : 0u) << (4 * (2 * jp + qh) + 2 * i + e);
    }
  }
  return z;
}

template <bool HAS_MASK, bool DROP>
__global__ void __launch_bounds__(BWD_THREADS, 1)
attn_bwd_kernel(const __grid_constant__ CUtensorMap tm_kv, const __grid_constant__ CUtensorMap tm_q,
                const __grid_constant__ CUtensorMap tm_do, const AttnDev p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sK = smem;
  uint8_t* sV = smem + 16384;
  uint8_t* sQd = smem + 32768;   // [2] x { Q chunk 8 KB, dO chunk 8 KB }
  uint8_t* sdST = smem + 65536;  // dS'^T [128 keys][64 q] bf16, 128B-swizzled
  float* s_nlse = reinterpret_cast<float*>(smem + 81920);  // [2][64]  -lse * log2(e)
  float* s_dsum = s_nlse + 2 * BQ;                          // [2][64]
  uint32_t* s_mask = reinterpret_cast<uint32_t*>(s_dsum + 2 * BQ);  // [MAX_MASK_WORDS] query validity bits
  uint64_t* bars = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(s_mask) + 512);
  uint64_t *bar_kv = bars, *bar_q = bars + 1 /* [2] */;

  const int tid = threadIdx.x, lane = tid & 31;
  const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);
  const int wg = warp >> 2, wq = warp & 3;
  const int kt = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  pdl_launch_dependents();
  const int S = p.S, H = p.H;
  const int k0 = kt * AT_N, tok0 = b * S;
  const int n_q = (S + BQ - 1) / BQ;

  if (tid == 0) {
    tma_prefetch_desc(&tm_kv); tma_prefetch_desc(&tm_q); tma_prefetch_desc(&tm_do);
    mbar_init(bar_kv, 1); mbar_init(&bar_q[0], 1); mbar_init(&bar_q[1], 1);
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();
  auto load_q = [&](int c) {
    uint8_t* buf = sQd + (c & 1) * 16384;
    mbar_arrive_expect_tx(&bar_q[c & 1], 16384);
    tma_load_2d(buf, &tm_q, &bar_q[c & 1], h * AT_D, tok0 + c * BQ);
    tma_load_2d(buf + 8192, &tm_do, &bar_q[c & 1], h * AT_D, tok0 + c * BQ);
  };
  if (tid == 0) {
    mbar_arrive_expect_tx(bar_kv, 32768);
    tma_load_2d(sK, &tm_kv, bar_kv, H + h * AT_D, tok0 + k0);
    tma_load_2d(sV, &tm_kv, bar_kv, 2 * H + h * AT_D, tok0 + k0);
    load_q(0);
    if (n_q > 1) load_q(1);
  }
  const size_t st0 = ((size_t)b * p.heads + h) * S;
  auto stage_stats = [&](int c) {  // threads 0..63
    const int q = c * BQ + tid;
    s_nlse[(c & 1) * BQ + tid] = (q < S) ? -p.lse[st0 + q] * LOG2E : 0.f;
    s_dsum[(c & 1) * BQ + tid] = (q < S) ? p.dsum[st0 + q] : 0.f;
  };
  if (tid < BQ) stage_stats(0);
  if (HAS_MASK) build_mask(s_mask, p.valid + tok0, n_q * BQ, S);
  __syncthreads();

  // this thread's two key rows (i = 0, 1)
  bool k_in[2], vk[2];
  int pair_lo[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int kk = k0 + wg * 64 + wq * 16 + (lane >> 2) + 8 * i;
    k_in[i] = kk < S;
    vk[i] = k_in[i] ? (HAS_MASK ? p.valid[tok0 + kk] != 0 : true) : false;
    pair_lo[i] = HAS_MASK ? pair_lo_of(kk, p.pair_P, p.pair_chunk) : -1;  // queries this key is seen by
  }
  const float sc2 = p.scale * LOG2E;
  float dv[32], dk[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) { dv[i] = 0.f; dk[i] = 0.f; }
  uint64_t drop_n16 = 0, drop_bh = 0, drop_key = 0;
  if (DROP) {
    drop_n16 = (uint64_t)((S + 15) >> 4);
    drop_bh = ((uint64_t)b * p.heads + h) * drop_n16;
    drop_key = (uint64_t)((k0 + wg * 64 + wq * 16) >> 4) * 8 + (lane >> 2);
  }

  mbar_wait(bar_kv, 0);
  const uint32_t ka = smem_u32(sK) + wg * 8192, va = smem_u32(sV) + wg * 8192;
  const uint32_t dsa = smem_u32(sdST);
  for (int c = 0; c < n_q; ++c) {
    const int bb = c & 1, q0 = c * BQ;
    mbar_wait(&bar_q[bb], (uint32_t)((c >> 1) & 1));
    const uint32_t qa = smem_u32(sQd + bb * 16384), da = qa + 8192;
    float s[32], dp[32];
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < AT_D / 16; ++k) wgmma_m64n64_ss<0, 0>(s, desc_kmajor(ka, k), desc_kmajor(qa, k), k > 0 ? 1u : 0u);
#pragma unroll
    for (int k = 0; k < AT_D / 16; ++k) wgmma_m64n64_ss<0, 0>(dp, desc_kmajor(va, k), desc_kmajor(da, k), k > 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(s);
    reg_fence(dp);
    const float* nlse = s_nlse + bb * BQ;
    const float* dsm = s_dsum + bb * BQ;
    uint32_t iw[2], qw[2];
#pragma unroll
    for (int w = 0; w < 2; ++w) {
      iw[w] = range_word(q0 + 32 * w, S);                                  // query in range
      qw[w] = HAS_MASK ? s_mask[(q0 >> 5) + w] : 0xffffffffu;              // query validity
    }
    const uint32_t zk = DROP ? attn_keep_bits_keyrows(p, drop_bh, drop_key, drop_n16, q0, lane) : 0u;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      uint32_t aw[2];
#pragma unroll
      for (int w = 0; w < 2; ++w)
        aw[w] = (HAS_MASK && pair_lo[i] >= 0) ? pair_word(q0 + 32 * w, pair_lo[i], p.pair_P, p.pair_chunk) : 0xffffffffu;
      const int row = wg * 64 + wq * 16 + (lane >> 2) + 8 * i;  // key row inside the tile
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
        float pv[2], dsv[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int col = 8 * jj + 2 * (lane & 3) + e, bit = col & 31, w = jj >> 2;
          float t = s[4 * jj + 2 * i + e] * sc2;
          t = (vk[i] && ((aw[w] >> bit) & 1u)) ? t : MASKED_LOG2;
          t = ((qw[w] >> bit) & 1u) ? t : 0.f;  // padding query: uniform row (zero scores)
          float pr = ex2_approx(t + nlse[col]);
          pr = (k_in[i] && ((iw[w] >> bit) & 1u)) ? pr : 0.f;
          // d(score)/d(q k^T) = m * scale (utils/transformer.py:109-110: scores*m - 1e10*(1-m)): a padding QUERY row keeps
          // its uniform probabilities for dV but sends nothing back into q and k.  (scale itself: dK epilogue / dQ finish)
          const float gq = ((qw[w] >> bit) & 1u) ? pr : 0.f;
          if (DROP) {  // dV += (P o Z s) dO;  dS' = P o (Z s dP - D)
            const float zs = ((zk >> (4 * jj + 2 * i + e)) & 1u) ? p.drop_scale : 0.f;
            pv[e] = pr * zs;
            dsv[e] = (dp[4 * jj + 2 * i + e] * zs - dsm[col]) * gq;
          } else {
            pv[e] = pr;
            dsv[e] = (dp[4 * jj + 2 * i + e] - dsm[col]) * gq;
          }
        }
        s[4 * jj + 2 * i] = pv[0]; s[4 * jj + 2 * i + 1] = pv[1];
        dp[4 * jj + 2 * i] = dsv[0]; dp[4 * jj + 2 * i + 1] = dsv[1];
        *reinterpret_cast<uint32_t*>(sdST + row * 128 + ((jj ^ (row & 7)) << 4) + (lane & 3) * 4) = pack_bf16x2(dsv[0], dsv[1]);
      }
    }
    // ---- dV += P^T dO, dK += dS'^T Q (A from registers; dO / Q MN-major: rows are queries) ----
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < BQ / 16; ++kk) {
      uint32_t a[4];
      acc_to_afrag(s, kk, a);
      wgmma_m64n64_rs<1>(dv, a, desc_mnmajor(da, kk, 0), 1u);
    }
#pragma unroll
    for (int kk = 0; kk < BQ / 16; ++kk) {
      uint32_t a[4];
      acc_to_afrag(dp, kk, a);
      wgmma_m64n64_rs<1>(dk, a, desc_mnmajor(qa, kk, 0), 1u);
    }
    wgmma_commit();
    fence_proxy_async_smem();                     // dS'^T (generic stores) -> wgmma operand reads
    asm volatile("bar.sync 1, 256;" ::: "memory");  // both warpgroups' halves of dS'^T are in place
    // ---- dQ_chunk[:, 32 wg : 32 wg + 32] = dS' K  (A = dS' as the MN-major view of dS'^T, B = K MN-major; over 128 keys) ----
    float dq[16];
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < AT_N / 16; ++k)
      wgmma_m64n32_ss<1, 1>(dq, desc_mnmajor(dsa, k, 0), desc_mnmajor(smem_u32(sK) + wg * 64, k, 0), k > 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(dv);
    reg_fence(dk);
    reg_fence(dq);
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int q = q0 + wq * 16 + (lane >> 2) + 8 * i;
      if (q >= S) continue;
      float* dst = p.dq_accum + (size_t)(tok0 + q) * p.ld_dq + h * AT_D + wg * 32 + 2 * (lane & 3);
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
        const float v0 = dq[4 * jj + 2 * i], v1 = dq[4 * jj + 2 * i + 1];
        asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(dst + 8 * jj), "f"(v0), "f"(v1) : "memory");
      }
    }
    if (tid < BQ && c + 1 < n_q) stage_stats(c + 1);  // buffer (c + 1) & 1 was last read by chunk c - 1
    __syncthreads();  // Q/dO buffer bb and dS'^T are free
    if (tid == 0 && c + 2 < n_q) load_q(c + 2);
  }
  // ---- dK (x 1/sqrt(d)), dV of this key tile (exclusive rows) ----
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int key = k0 + wg * 64 + wq * 16 + (lane >> 2) + 8 * i;
    if (key >= S) continue;
    bf16* dst = p.dqkv + (size_t)(tok0 + key) * p.ld_dqkv + h * AT_D + 2 * (lane & 3);
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) {
      *reinterpret_cast<uint32_t*>(dst + H + 8 * jj) = pack_bf16x2(dk[4 * jj + 2 * i] * p.scale, dk[4 * jj + 2 * i + 1] * p.scale);
      *reinterpret_cast<uint32_t*>(dst + 2 * H + 8 * jj) = pack_bf16x2(dv[4 * jj + 2 * i], dv[4 * jj + 2 * i + 1]);
    }
  }
}

// D[b,h,q] = sum_d dO[q,hd] * O[q,hd]   (one warp per (token, head) pair would waste lanes; 8 lanes x 8 elems per head)
__global__ void attn_dsum_kernel(const bf16* __restrict__ o, const bf16* __restrict__ d_o, int ld, float* __restrict__ dsum,
                                 int B, int S, int heads) {
  pdl_launch_dependents();
  pdl_wait();
  const long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long item = gid >> 3;  // (token, head)
  const int sub = (int)(gid & 7);
  const long long total = (long long)B * S * heads;
  float acc = 0.f;
  if (item < total) {
    const int hh = (int)(item % heads);
    const long long tok = item / heads;
    const size_t off = (size_t)tok * ld + hh * AT_D + sub * 8;
    uint4 a = __ldg(reinterpret_cast<const uint4*>(o + off));
    uint4 g = __ldg(reinterpret_cast<const uint4*>(d_o + off));
    const uint32_t* pa = reinterpret_cast<const uint32_t*>(&a);
    const uint32_t* pg = reinterpret_cast<const uint32_t*>(&g);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float2 x = unpack_bf16x2(pa[i]), y = unpack_bf16x2(pg[i]);
      acc += x.x * y.x + x.y * y.y;
    }
  }
  acc += __shfl_xor_sync(0xffffffffu, acc, 1);
  acc += __shfl_xor_sync(0xffffffffu, acc, 2);
  acc += __shfl_xor_sync(0xffffffffu, acc, 4);
  if (item < total && sub == 0) {
    const int hh = (int)(item % heads);
    const long long tok = item / heads;
    const int bb = (int)(tok / S), q = (int)(tok % S);
    dsum[((size_t)bb * heads + hh) * S + q] = acc;
  }
}

// dq fp32 accumulator -> bf16 q-block of dqkv (and re-zero the accumulator for the next layer), fused with the column sums
// of the whole dqkv row block = the gradient of the fused q/k/v bias.  grid = (ceil(3H/256), row slabs), 8 warps, lane = 8 cols.
__global__ void __launch_bounds__(256) attn_dqkv_finish_kernel(float* __restrict__ dq, int ld_dq, bf16* __restrict__ dqkv, int ld_dqkv,
                                                               long long rows, int H, float* __restrict__ bias_grad, float scale) {
  __shared__ float sred[8][256];
  pdl_launch_dependents();
  pdl_wait();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int col = blockIdx.x * 256 + lane * 8;
  float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  if (col < 3 * H) {
    for (long long r = (long long)blockIdx.y * 8 + warp; r < rows; r += (long long)gridDim.y * 8) {
      float v[8];
      bf16* o = dqkv + (size_t)r * ld_dqkv + col;
      if (col < H) {
        float4* src = reinterpret_cast<float4*>(dq + (size_t)r * ld_dq + col);
        const float4 a = src[0], b = src[1];
        src[0] = make_float4(0.f, 0.f, 0.f, 0.f);
        src[1] = make_float4(0.f, 0.f, 0.f, 0.f);
        // K3 accumulates dS' K without the 1/sqrt(d) of the scores: applied here, once per output element
        const uint4 pk = make_uint4(pack_bf16x2(a.x * scale, a.y * scale), pack_bf16x2(a.z * scale, a.w * scale),
                                    pack_bf16x2(b.x * scale, b.y * scale), pack_bf16x2(b.z * scale, b.w * scale));
        *reinterpret_cast<uint4*>(o) = pk;
        const uint32_t* pu = reinterpret_cast<const uint32_t*>(&pk);
#pragma unroll
        for (int i = 0; i < 4; ++i) { const float2 f = unpack_bf16x2(pu[i]); v[2 * i] = f.x; v[2 * i + 1] = f.y; }
      } else {
        const uint4 u = *reinterpret_cast<const uint4*>(o);
        const uint32_t* pu = reinterpret_cast<const uint32_t*>(&u);
#pragma unroll
        for (int i = 0; i < 4; ++i) { const float2 f = unpack_bf16x2(pu[i]); v[2 * i] = f.x; v[2 * i + 1] = f.y; }
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] += v[i];
    }
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) sred[warp][lane * 8 + i] = acc[i];
  __syncthreads();
  const int c = threadIdx.x;
  if (bias_grad != nullptr && blockIdx.x * 256 + c < 3 * H) {
    float s2 = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) s2 += sred[w][c];
    atomicAdd(bias_grad + blockIdx.x * 256 + c, s2);
  }
}

// -----------------------------------------------------------------------------------------------------------------
// backward for sequences of <= 512 tokens: a dQ kernel (queries on the accumulator rows) launched first, then a dK/dV kernel
// (keys on the rows).  Both recompute S and dP, which costs 1.4x K3's tensor work, and in return neither needs anything from
// the other CTAs of its grid: no fp32 dQ workspace, no finish pass, no dsum pass, no atomics except one per bias column.
// Each CTA is one warpgroup owning a 64-row tile, so a short sequence pads its last tile to 64 rows (not 128 as K3 does),
// and two or three CTAs share an SM: one CTA's softmax runs under another's wgmma.  The mask, padding-query and dropout rules
// are K3's, element for element; both orientations draw the same dropout bits (ptx.cuh attn_dropout_words).
// -----------------------------------------------------------------------------------------------------------------
constexpr int SB_THREADS = 128;   // one warpgroup
constexpr int SB_ROWS = 64;       // query rows (dQ kernel) / key rows (dK/dV kernel) per CTA
constexpr int SB_MASK_WORDS = 16; // validity bits of 512 positions
// Q, dO, O (8 KB each), 2 x {K, V} chunk (8 KB each), bias column partials [4][64], -lse log2(e) and D [2][64], key mask,
// barriers, alignment
constexpr int DQ_SMEM = 3 * 8192 + 2 * 16384 + 1024 + 512 + 64 + 64 + 1024;
// K, V (8 KB each), 2 x {Q, dO} chunk (8 KB each), bias column partials [2][4][64], statistics [2][2][64], query mask,
// barriers, alignment
constexpr int DKV_SMEM = 2 * 8192 + 2 * 16384 + 2048 + 1024 + 64 + 64 + 1024;

// dQ of 64 queries of one (b, h): D = rowsum(dO o O) from the TMA-loaded O and dO tiles (written to dsum for the dK/dV kernel),
// then 64-key chunks of K and V through a two-buffer TMA ring:
//   S = Q K^T, dP = dO V^T                     (wgmma, smem x smem)
//   P = exp2(S sc - lse), dS' = P (dP - D)     (registers; a padding query row sends nothing into dQ)
//   dQ += dS' K                                (wgmma, A = dS' straight from registers, K MN-major)
// and dQ x 1/sqrt(d) goes to the q block of dqkv as bf16.
template <bool HAS_MASK, bool DROP>
__global__ void __launch_bounds__(SB_THREADS, 3)
attn_bwd_dq_kernel(const __grid_constant__ CUtensorMap tm_qkv, const __grid_constant__ CUtensorMap tm_do,
                   const __grid_constant__ CUtensorMap tm_o, const AttnDev p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;
  uint8_t* sdO = smem + 8192;
  uint8_t* sO = smem + 16384;
  uint8_t* sKV = smem + 24576;  // [2] x { K chunk 8 KB, V chunk 8 KB }: chunk j lives in buffer j & 1
  float* s_red = reinterpret_cast<float*>(smem + 57344);  // [4][64]
  float* s_nlse = s_red + 256;                            // [64]  -lse * log2(e)
  float* s_dsum = s_nlse + SB_ROWS;                       // [64]
  uint32_t* s_mask = reinterpret_cast<uint32_t*>(s_dsum + SB_ROWS);  // [SB_MASK_WORDS] key validity bits
  uint64_t* bars = reinterpret_cast<uint64_t*>(s_mask + SB_MASK_WORDS);
  uint64_t *bar_q = bars, *bar_kv = bars + 1 /* [2] */;

  const int tid = threadIdx.x, lane = tid & 31;
  const int wq = __shfl_sync(0xffffffffu, tid >> 5, 0);
  const int q0 = blockIdx.x * SB_ROWS, h = blockIdx.y, b = blockIdx.z;
  pdl_launch_dependents();
  const int S = p.S, H = p.H, tok0 = b * S;
  const int n_kv = (S + SB_ROWS - 1) / SB_ROWS;

  if (tid == 0) {
    tma_prefetch_desc(&tm_qkv); tma_prefetch_desc(&tm_do); tma_prefetch_desc(&tm_o);
    mbar_init(bar_q, 1); mbar_init(&bar_kv[0], 1); mbar_init(&bar_kv[1], 1);
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();
  auto load_kv = [&](int j) {
    uint8_t* buf = sKV + (j & 1) * 16384;
    mbar_arrive_expect_tx(&bar_kv[j & 1], 16384);
    tma_load_2d(buf, &tm_qkv, &bar_kv[j & 1], H + h * AT_D, tok0 + j * SB_ROWS);
    tma_load_2d(buf + 8192, &tm_qkv, &bar_kv[j & 1], 2 * H + h * AT_D, tok0 + j * SB_ROWS);
  };
  if (tid == 0) {
    mbar_arrive_expect_tx(bar_q, 3 * 8192);
    tma_load_2d(sQ, &tm_qkv, bar_q, h * AT_D, tok0 + q0);
    tma_load_2d(sdO, &tm_do, bar_q, h * AT_D, tok0 + q0);
    tma_load_2d(sO, &tm_o, bar_q, h * AT_D, tok0 + q0);
    load_kv(0);
    if (n_kv > 1) load_kv(1);
  }
  const size_t st0 = ((size_t)b * p.heads + h) * S;
  if (tid < SB_ROWS) s_nlse[tid] = (q0 + tid < S) ? -p.lse[st0 + q0 + tid] * LOG2E : 0.f;
  if (HAS_MASK) build_mask(s_mask, p.valid + tok0, n_kv * SB_ROWS, S);
  mbar_wait(bar_q, 0);
  // D: 8 lanes per query row, 8 columns each, summed in the order of attn_dsum_kernel (the long-sequence path)
#pragma unroll
  for (int it = 0; it < 4; ++it) {
    const int r = it * 16 + (tid >> 3), sub = tid & 7;
    const uint4 a = *reinterpret_cast<const uint4*>(sO + sw128_offset(r, sub));
    const uint4 g = *reinterpret_cast<const uint4*>(sdO + sw128_offset(r, sub));
    const uint32_t* pa = reinterpret_cast<const uint32_t*>(&a);
    const uint32_t* pg = reinterpret_cast<const uint32_t*>(&g);
    float acc = 0.f;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float2 x = unpack_bf16x2(pa[i]), y = unpack_bf16x2(pg[i]);
      acc += x.x * y.x + x.y * y.y;
    }
    acc += __shfl_xor_sync(0xffffffffu, acc, 1);
    acc += __shfl_xor_sync(0xffffffffu, acc, 2);
    acc += __shfl_xor_sync(0xffffffffu, acc, 4);
    if (sub == 0) {
      s_dsum[r] = acc;
      if (q0 + r < S) p.dsum[st0 + q0 + r] = acc;
    }
  }
  __syncthreads();

  // this thread's two query rows (i = 0, 1); gq: the row is in range and valid, so it sends its gradient into q and k
  float nl[2], dd[2];
  bool gq[2];
  int pair_lo[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int r = wq * 16 + (lane >> 2) + 8 * i, q = q0 + r;
    nl[i] = s_nlse[r];
    dd[i] = s_dsum[r];
    const bool vq = (HAS_MASK && q < S) ? (p.valid[tok0 + q] != 0) : true;
    gq[i] = q < S && vq;
    pair_lo[i] = (HAS_MASK && vq) ? pair_lo_of(q, p.pair_P, p.pair_chunk) : -1;  // keys this query may see
  }
  const float sc2 = p.scale * LOG2E;
  float dq[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) dq[i] = 0.f;
  uint64_t drop_row = 0;
  if (DROP) {
    const uint64_t n16 = (uint64_t)((S + 15) >> 4);
    drop_row = ((((uint64_t)b * p.heads + h) * n16 + (uint64_t)((q0 + wq * 16) >> 4)) * 8 + (lane >> 2)) * n16 * 8;
  }
  const uint32_t qa = smem_u32(sQ), da = smem_u32(sdO);
  for (int j = 0; j < n_kv; ++j) {
    const int k0 = j * SB_ROWS;
    const uint32_t zq = DROP ? attn_keep_bits_queryrows(p, drop_row, k0, lane) : 0u;
    mbar_wait(&bar_kv[j & 1], (uint32_t)((j >> 1) & 1));
    const uint32_t ka = smem_u32(sKV + (j & 1) * 16384), va = ka + 8192;
    float s[32], dp[32];
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < AT_D / 16; ++k) wgmma_m64n64_ss<0, 0>(s, desc_kmajor(qa, k), desc_kmajor(ka, k), k > 0 ? 1u : 0u);
#pragma unroll
    for (int k = 0; k < AT_D / 16; ++k) wgmma_m64n64_ss<0, 0>(dp, desc_kmajor(da, k), desc_kmajor(va, k), k > 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(s);
    reg_fence(dp);
    uint32_t iw[2], kw[2];
#pragma unroll
    for (int w = 0; w < 2; ++w) {
      iw[w] = range_word(k0 + 32 * w, S);                           // key in range
      kw[w] = HAS_MASK ? s_mask[(k0 >> 5) + w] : 0xffffffffu;       // key validity
    }
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      uint32_t aw[2];
#pragma unroll
      for (int w = 0; w < 2; ++w)
        aw[w] = kw[w] & ((HAS_MASK && pair_lo[i] >= 0) ? pair_word(k0 + 32 * w, pair_lo[i], p.pair_P, p.pair_chunk) : 0xffffffffu);
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int x = 4 * jj + 2 * i + e, bit = (8 * jj + 2 * (lane & 3) + e) & 31, w = jj >> 2;
          float t = s[x] * sc2;
          t = ((aw[w] >> bit) & 1u) ? t : MASKED_LOG2;
          float pr = ex2_approx(t + nl[i]);
          pr = (gq[i] && ((iw[w] >> bit) & 1u)) ? pr : 0.f;
          if (DROP) {
            const float zs = ((zq >> x) & 1u) ? p.drop_scale : 0.f;
            dp[x] = (dp[x] * zs - dd[i]) * pr;
          } else {
            dp[x] = (dp[x] - dd[i]) * pr;
          }
        }
      }
    }
    // ---- dQ += dS' K (A from registers; K MN-major: rows are keys) ----
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < SB_ROWS / 16; ++kk) {
      uint32_t a[4];
      acc_to_afrag(dp, kk, a);
      wgmma_m64n64_rs<1>(dq, a, desc_mnmajor(ka, kk, 0), 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(dq);
    __syncthreads();  // buffer j & 1 is free
    if (tid == 0 && j + 2 < n_kv) load_kv(j + 2);
  }
  // ---- dQ x 1/sqrt(d) -> bf16 q block; the bias column sums take the rounded values ----
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int q = q0 + wq * 16 + (lane >> 2) + 8 * i;
    bf16* dst = p.dqkv + (size_t)(tok0 + q) * p.ld_dqkv + h * AT_D + 2 * (lane & 3);
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) {
      const uint32_t u = pack_bf16x2(dq[4 * jj + 2 * i] * p.scale, dq[4 * jj + 2 * i + 1] * p.scale);
      const float2 f = unpack_bf16x2(u);
      dq[4 * jj + 2 * i] = q < S ? f.x : 0.f;
      dq[4 * jj + 2 * i + 1] = q < S ? f.y : 0.f;
      if (q < S) *reinterpret_cast<uint32_t*>(dst + 8 * jj) = u;
    }
  }
  if (p.d_bias) bias_colsum_add(dq, s_red, p.d_bias + h * AT_D, wq, lane, tid);
}

// dK and dV of 64 keys of one (b, h): K3 without its dQ half.  64-query chunks of Q and dO through a two-buffer TMA ring, with
// the chunk's -lse log2(e) and D (written by attn_bwd_dq_kernel) staged in smem.  Per chunk:
//   S^T = K Q^T, dP^T = V dO^T                       (wgmma, smem x smem)
//   P^T = exp2(S^T sc - lse), dS'^T = P^T (dP^T - D)  (registers)
//   dV += P^T dO, dK += dS'^T Q                        (wgmma, A straight from registers, dO / Q MN-major)
template <bool HAS_MASK, bool DROP>
__global__ void __launch_bounds__(SB_THREADS, 2)
attn_bwd_dkdv_kernel(const __grid_constant__ CUtensorMap tm_qkv, const __grid_constant__ CUtensorMap tm_do, const AttnDev p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sK = smem;
  uint8_t* sV = smem + 8192;
  uint8_t* sQd = smem + 16384;  // [2] x { Q chunk 8 KB, dO chunk 8 KB }
  float* s_red = reinterpret_cast<float*>(smem + 49152);  // [2][4][64]
  float* s_nlse = s_red + 512;                            // [2][64]  -lse * log2(e)
  float* s_dsum = s_nlse + 2 * BQ;                        // [2][64]
  uint32_t* s_mask = reinterpret_cast<uint32_t*>(s_dsum + 2 * BQ);  // [SB_MASK_WORDS] query validity bits
  uint64_t* bars = reinterpret_cast<uint64_t*>(s_mask + SB_MASK_WORDS);
  uint64_t *bar_kv = bars, *bar_q = bars + 1 /* [2] */;

  const int tid = threadIdx.x, lane = tid & 31;
  const int wq = __shfl_sync(0xffffffffu, tid >> 5, 0);
  const int k0 = blockIdx.x * SB_ROWS, h = blockIdx.y, b = blockIdx.z;
  pdl_launch_dependents();
  const int S = p.S, H = p.H, tok0 = b * S;
  const int n_q = (S + BQ - 1) / BQ;

  if (tid == 0) {
    tma_prefetch_desc(&tm_qkv); tma_prefetch_desc(&tm_do);
    mbar_init(bar_kv, 1); mbar_init(&bar_q[0], 1); mbar_init(&bar_q[1], 1);
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();  // before the first read of dsum: the dQ kernel writes it
  auto load_q = [&](int c) {
    uint8_t* buf = sQd + (c & 1) * 16384;
    mbar_arrive_expect_tx(&bar_q[c & 1], 16384);
    tma_load_2d(buf, &tm_qkv, &bar_q[c & 1], h * AT_D, tok0 + c * BQ);
    tma_load_2d(buf + 8192, &tm_do, &bar_q[c & 1], h * AT_D, tok0 + c * BQ);
  };
  if (tid == 0) {
    mbar_arrive_expect_tx(bar_kv, 16384);
    tma_load_2d(sK, &tm_qkv, bar_kv, H + h * AT_D, tok0 + k0);
    tma_load_2d(sV, &tm_qkv, bar_kv, 2 * H + h * AT_D, tok0 + k0);
    load_q(0);
    if (n_q > 1) load_q(1);
  }
  const size_t st0 = ((size_t)b * p.heads + h) * S;
  auto stage_stats = [&](int c) {  // threads 0..63
    const int q = c * BQ + tid;
    s_nlse[(c & 1) * BQ + tid] = (q < S) ? -p.lse[st0 + q] * LOG2E : 0.f;
    s_dsum[(c & 1) * BQ + tid] = (q < S) ? p.dsum[st0 + q] : 0.f;
  };
  if (tid < BQ) stage_stats(0);
  if (HAS_MASK) build_mask(s_mask, p.valid + tok0, n_q * BQ, S);
  __syncthreads();

  // this thread's two key rows (i = 0, 1)
  bool k_in[2], vk[2];
  int pair_lo[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int kk = k0 + wq * 16 + (lane >> 2) + 8 * i;
    k_in[i] = kk < S;
    vk[i] = k_in[i] ? (HAS_MASK ? p.valid[tok0 + kk] != 0 : true) : false;
    pair_lo[i] = HAS_MASK ? pair_lo_of(kk, p.pair_P, p.pair_chunk) : -1;  // queries this key is seen by
  }
  const float sc2 = p.scale * LOG2E;
  float dv[32], dk[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) { dv[i] = 0.f; dk[i] = 0.f; }
  uint64_t drop_n16 = 0, drop_bh = 0, drop_key = 0;
  if (DROP) {
    drop_n16 = (uint64_t)((S + 15) >> 4);
    drop_bh = ((uint64_t)b * p.heads + h) * drop_n16;
    drop_key = (uint64_t)((k0 + wq * 16) >> 4) * 8 + (lane >> 2);
  }

  mbar_wait(bar_kv, 0);
  const uint32_t ka = smem_u32(sK), va = smem_u32(sV);
  for (int c = 0; c < n_q; ++c) {
    const int bb = c & 1, q0 = c * BQ;
    const uint32_t zk = DROP ? attn_keep_bits_keyrows(p, drop_bh, drop_key, drop_n16, q0, lane) : 0u;
    mbar_wait(&bar_q[bb], (uint32_t)((c >> 1) & 1));
    const uint32_t qa = smem_u32(sQd + bb * 16384), da = qa + 8192;
    float s[32], dp[32];
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < AT_D / 16; ++k) wgmma_m64n64_ss<0, 0>(s, desc_kmajor(ka, k), desc_kmajor(qa, k), k > 0 ? 1u : 0u);
#pragma unroll
    for (int k = 0; k < AT_D / 16; ++k) wgmma_m64n64_ss<0, 0>(dp, desc_kmajor(va, k), desc_kmajor(da, k), k > 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(s);
    reg_fence(dp);
    const float* nlse = s_nlse + bb * BQ;
    const float* dsm = s_dsum + bb * BQ;
    uint32_t iw[2], qw[2];
#pragma unroll
    for (int w = 0; w < 2; ++w) {
      iw[w] = range_word(q0 + 32 * w, S);                                  // query in range
      qw[w] = HAS_MASK ? s_mask[(q0 >> 5) + w] : 0xffffffffu;              // query validity
    }
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      uint32_t aw[2];
#pragma unroll
      for (int w = 0; w < 2; ++w)
        aw[w] = (HAS_MASK && pair_lo[i] >= 0) ? pair_word(q0 + 32 * w, pair_lo[i], p.pair_P, p.pair_chunk) : 0xffffffffu;
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int x = 4 * jj + 2 * i + e, col = 8 * jj + 2 * (lane & 3) + e, bit = col & 31, w = jj >> 2;
          float t = s[x] * sc2;
          t = (vk[i] && ((aw[w] >> bit) & 1u)) ? t : MASKED_LOG2;
          t = ((qw[w] >> bit) & 1u) ? t : 0.f;  // padding query: uniform row (zero scores)
          float pr = ex2_approx(t + nlse[col]);
          pr = (k_in[i] && ((iw[w] >> bit) & 1u)) ? pr : 0.f;
          const float gq = ((qw[w] >> bit) & 1u) ? pr : 0.f;  // a padding query keeps P for dV, sends nothing into k
          if (DROP) {
            const float zs = ((zk >> x) & 1u) ? p.drop_scale : 0.f;
            s[x] = pr * zs;
            dp[x] = (dp[x] * zs - dsm[col]) * gq;
          } else {
            s[x] = pr;
            dp[x] = (dp[x] - dsm[col]) * gq;
          }
        }
      }
    }
    // ---- dV += P^T dO, dK += dS'^T Q (A from registers; dO / Q MN-major: rows are queries) ----
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < BQ / 16; ++kk) {
      uint32_t a[4];
      acc_to_afrag(s, kk, a);
      wgmma_m64n64_rs<1>(dv, a, desc_mnmajor(da, kk, 0), 1u);
    }
#pragma unroll
    for (int kk = 0; kk < BQ / 16; ++kk) {
      uint32_t a[4];
      acc_to_afrag(dp, kk, a);
      wgmma_m64n64_rs<1>(dk, a, desc_mnmajor(qa, kk, 0), 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(dv);
    reg_fence(dk);
    if (tid < BQ && c + 1 < n_q) stage_stats(c + 1);  // buffer (c + 1) & 1 was last read by chunk c - 1
    __syncthreads();  // Q/dO buffer bb is free
    if (tid == 0 && c + 2 < n_q) load_q(c + 2);
  }
  // ---- dK (x 1/sqrt(d)), dV of this key tile; the bias column sums take the rounded values ----
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int key = k0 + wq * 16 + (lane >> 2) + 8 * i;
    bf16* dst = p.dqkv + (size_t)(tok0 + key) * p.ld_dqkv + h * AT_D + 2 * (lane & 3);
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) {
      const int x = 4 * jj + 2 * i;
      const uint32_t uk = pack_bf16x2(dk[x] * p.scale, dk[x + 1] * p.scale), uv = pack_bf16x2(dv[x], dv[x + 1]);
      const float2 fk = unpack_bf16x2(uk), fv = unpack_bf16x2(uv);
      dk[x] = key < S ? fk.x : 0.f; dk[x + 1] = key < S ? fk.y : 0.f;
      dv[x] = key < S ? fv.x : 0.f; dv[x + 1] = key < S ? fv.y : 0.f;
      if (key < S) {
        *reinterpret_cast<uint32_t*>(dst + H + 8 * jj) = uk;
        *reinterpret_cast<uint32_t*>(dst + 2 * H + 8 * jj) = uv;
      }
    }
  }
  if (p.d_bias) {
    bias_colsum_add(dk, s_red, p.d_bias + H + h * AT_D, wq, lane, tid);
    bias_colsum_add(dv, s_red + 256, p.d_bias + 2 * H + h * AT_D, wq, lane, tid);
  }
}

// -----------------------------------------------------------------------------------------------------------------
// K4: colsum[b,k] += (1/heads) * sum_q P[b,h,q,k], recomputed from (q,k,lse); keys on the accumulator rows so the reduction
// over queries runs along registers.  One CTA per (128-key tile, head, batch), warpgroup w owns keys [64 w, 64 w + 64); the
// query chunks of 64 run through a two-buffer TMA ring.
// -----------------------------------------------------------------------------------------------------------------
constexpr int CS_THREADS = 256;
constexpr int CS_SMEM = 16384 + 2 * 8192 + 512 + 512 + 64 + 1024;  // K, 2 x Q chunk, statistics, query mask, barriers, alignment

template <bool HAS_MASK, bool DROP>
__global__ void __launch_bounds__(CS_THREADS, 2) attn_colsum_kernel(const __grid_constant__ CUtensorMap tm_k, const __grid_constant__ CUtensorMap tm_q,
                                                                    const AttnDev p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sK = smem;
  uint8_t* sQ = smem + 16384;                                    // [2] x 8 KB
  float* s_nlse = reinterpret_cast<float*>(smem + 32768);        // [2][64]  -lse * log2(e)
  uint32_t* s_mask = reinterpret_cast<uint32_t*>(smem + 32768 + 512);  // query validity bits
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + 32768 + 1024);
  uint64_t *bar_k = bars, *bar_q = bars + 1 /* [2] */;
  const int tid = threadIdx.x, lane = tid & 31;
  const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);
  const int wg = warp >> 2, wq = warp & 3;
  const int k0 = blockIdx.x * AT_N, h = blockIdx.y, b = blockIdx.z;
  const int S = p.S, H = p.H, tok0 = b * S;
  const int n_q = (S + BQ - 1) / BQ;
  pdl_launch_dependents();
  if (tid == 0) {
    tma_prefetch_desc(&tm_k); tma_prefetch_desc(&tm_q);
    mbar_init(bar_k, 1); mbar_init(&bar_q[0], 1); mbar_init(&bar_q[1], 1);
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();
  auto load_q = [&](int c) {
    mbar_arrive_expect_tx(&bar_q[c & 1], 8192);
    tma_load_2d(sQ + (c & 1) * 8192, &tm_q, &bar_q[c & 1], h * AT_D, tok0 + c * BQ);
  };
  if (tid == 0) {
    mbar_arrive_expect_tx(bar_k, 16384);
    tma_load_2d(sK, &tm_k, bar_k, H + h * AT_D, tok0 + k0);
    load_q(0);
    if (n_q > 1) load_q(1);
  }
  auto stage_lse = [&](int c) {  // threads 0..63
    const int q = c * BQ + tid;
    s_nlse[(c & 1) * BQ + tid] = (q < S) ? -p.lse[((size_t)b * p.heads + h) * S + q] * LOG2E : 0.f;
  };
  if (tid < BQ) stage_lse(0);
  if (HAS_MASK) build_mask(s_mask, p.valid + tok0, n_q * BQ, S);
  __syncthreads();

  bool k_in[2], vk[2];
  int pair_lo[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int kk = k0 + wg * 64 + wq * 16 + (lane >> 2) + 8 * i;
    k_in[i] = kk < S;
    vk[i] = k_in[i] ? (HAS_MASK ? p.valid[tok0 + kk] != 0 : true) : false;
    pair_lo[i] = HAS_MASK ? pair_lo_of(kk, p.pair_P, p.pair_chunk) : -1;  // queries this key is seen by
  }
  const float sc2 = p.scale * LOG2E;
  const int split = p.colsum2 ? p.colsum_split : 0x7fffffff;
  float acc[2] = {0.f, 0.f}, acc2[2] = {0.f, 0.f};
  uint64_t drop_n16 = 0, drop_bh = 0, drop_key = 0;
  if (DROP) {
    drop_n16 = (uint64_t)((S + 15) >> 4);
    drop_bh = ((uint64_t)b * p.heads + h) * drop_n16;
    drop_key = (uint64_t)((k0 + wg * 64 + wq * 16) >> 4) * 8 + (lane >> 2);
  }
  mbar_wait(bar_k, 0);
  const uint32_t ka = smem_u32(sK) + wg * 8192;
  for (int c = 0; c < n_q; ++c) {
    const int q0 = c * BQ;
    mbar_wait(&bar_q[c & 1], (uint32_t)((c >> 1) & 1));
    const uint32_t qa = smem_u32(sQ + (c & 1) * 8192);
    float s[32];
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < AT_D / 16; ++k) wgmma_m64n64_ss<0, 0>(s, desc_kmajor(ka, k), desc_kmajor(qa, k), k > 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(s);
    const float* nl = s_nlse + (c & 1) * BQ;
    uint32_t qw[2], sw[2], iw[2];
#pragma unroll
    for (int w = 0; w < 2; ++w) {
      iw[w] = range_word(q0 + 32 * w, S);                              // query in range
      qw[w] = HAS_MASK ? s_mask[(q0 >> 5) + w] : 0xffffffffu;          // query validity
      sw[w] = range_word(q0 + 32 * w, split);                          // query < split -> colsum, else colsum2
    }
    const uint32_t zk = DROP ? attn_keep_bits_keyrows(p, drop_bh, drop_key, drop_n16, q0, lane) : 0u;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      uint32_t aw[2], keep[2];
#pragma unroll
      for (int w = 0; w < 2; ++w) {
        aw[w] = (HAS_MASK && pair_lo[i] >= 0) ? pair_word(q0 + 32 * w, pair_lo[i], p.pair_P, p.pair_chunk) : 0xffffffffu;
        keep[w] = (k_in[i] ? iw[w] : 0u) & ((HAS_MASK && p.colsum_valid_q) ? qw[w] : 0xffffffffu);  // queries that contribute at all
      }
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int col = 8 * jj + 2 * (lane & 3) + e, bit = col & 31, w = jj >> 2;
          float x = s[4 * jj + 2 * i + e] * sc2;
          x = (vk[i] && ((aw[w] >> bit) & 1u)) ? x : MASKED_LOG2;
          x = ((qw[w] >> bit) & 1u) ? x : 0.f;  // padding query: uniform row (zero scores)
          float pr = ex2_approx(x + nl[col]);
          pr = ((keep[w] >> bit) & 1u) ? pr : 0.f;
          if (DROP && !((zk >> (4 * jj + 2 * i + e)) & 1u)) pr = 0.f;  // P o Z; the scale s is applied once per sum below
          if ((sw[w] >> bit) & 1u) acc[i] += pr; else acc2[i] += pr;
        }
      }
    }
    if (tid < BQ && c + 1 < n_q) stage_lse(c + 1);  // buffer (c + 1) & 1 was last read by chunk c - 1
    __syncthreads();  // Q buffer c & 1 is free
    if (tid == 0 && c + 2 < n_q) load_q(c + 2);
  }
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    quad_sum(acc[i]);
    quad_sum(acc2[i]);
    if (DROP) { acc[i] *= p.drop_scale; acc2[i] *= p.drop_scale; }
    const int kk = k0 + wg * 64 + wq * 16 + (lane >> 2) + 8 * i;
    if ((lane & 3) == 0 && k_in[i]) {
      atomicAdd(p.colsum + (size_t)b * S + kk, acc[i] / (float)p.heads);
      if (p.colsum2) atomicAdd(p.colsum2 + (size_t)b * S + kk, acc2[i] / (float)p.heads);
    }
  }
}

static int check_common(const merlot_attn_t* a) {
  MB_REQUIRE(a != nullptr, MERLOT_EINVAL, "attention: null descriptor");
  MB_REQUIRE(a->B > 0 && a->S > 0 && a->heads > 0, MERLOT_ESHAPE, "attention: bad dims B=%d S=%d heads=%d", a->B, a->S,
             a->heads);
  MB_REQUIRE(a->head_dim == 64, MERLOT_ESHAPE, "attention: head size must be 64 (got %d)", a->head_dim);
  MB_REQUIRE(a->qkv != nullptr && a->ld_qkv >= 3 * a->heads * 64 && (a->ld_qkv % 8) == 0, MERLOT_ESHAPE,
             "attention: qkv must be [tokens, >=3H] with ld %% 8 == 0");
  MB_REQUIRE(a->pair_chunk_len >= 0 && a->pair_viz_len >= 0 && (a->pair_chunk_len == 0 || a->valid != nullptr), MERLOT_EINVAL,
             "attention: pair_chunk_len > 0 (disable_pairwise_lang_attn) needs the token-validity mask and non-negative lengths");
  MB_REQUIRE(a->dropout_p >= 0.f && a->dropout_p < 1.f, MERLOT_EINVAL, "attention: dropout_p must lie in [0, 1) (got %g)",
             (double)a->dropout_p);
  return MERLOT_OK;
}

static void fill_dev(const merlot_attn_t* a, AttnDev* p) {
  memset(p, 0, sizeof(*p));
  p->B = a->B; p->S = a->S; p->heads = a->heads; p->H = a->heads * 64;
  p->valid = reinterpret_cast<const uint8_t*>(a->valid);
  p->scale = a->scale;
  p->ctx = reinterpret_cast<bf16*>(a->ctx); p->ld_ctx = a->ld_ctx;
  p->lse = a->lse;
  p->dsum = a->dsum;
  p->dq_accum = a->dq_accum; p->ld_dq = a->ld_dq;
  p->dqkv = reinterpret_cast<bf16*>(a->dqkv); p->ld_dqkv = a->ld_dqkv;
  p->colsum = a->colsum;
  p->colsum2 = a->colsum2;
  p->colsum_split = a->colsum_split;
  p->colsum_valid_q = a->colsum_valid_q;
  p->pair_P = a->pair_viz_len; p->pair_chunk = a->pair_chunk_len;
  // the same float32 quantisation as the hidden-dropout kernels (gemm.cu, rowwise.cu)
  p->drop_thresh16 = (uint32_t)(a->dropout_p * 65536.0f + 0.5f);
  p->drop_scale = 1.0f / (1.0f - a->dropout_p);
  p->drop_seed = a->dropout_seed; p->drop_site = a->dropout_site;
}

}  // namespace mb

using namespace mb;

extern "C" int merlot_attention_fwd(const merlot_attn_t* a, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  int rc = check_common(a);
  if (rc) return rc;
  MB_REQUIRE(a->ctx != nullptr && (a->ld_ctx % 8) == 0, MERLOT_EINVAL, "attention_fwd: ctx missing or ld_ctx %% 8 != 0");
  AttnDev p; fill_dev(a, &p);
  CUtensorMap tq, tkv;
  rc = make_tmap_bf16_2d(&tq, a->qkv, (uint64_t)a->ld_qkv, (uint64_t)a->B * a->S, (uint64_t)a->ld_qkv, 64, AT_M);
  if (rc) return rc;
  rc = make_tmap_bf16_2d(&tkv, a->qkv, (uint64_t)a->ld_qkv, (uint64_t)a->B * a->S, (uint64_t)a->ld_qkv, 64, FK);
  if (rc) return rc;
  MB_REQUIRE(a->S <= MAX_MASK_WORDS * 32 - AT_N, MERLOT_ESHAPE, "attention_fwd: sequence longer than %d keys", MAX_MASK_WORDS * 32 - AT_N);
  static bool attr = false;
  if (!attr) {
    MB_CHECK_CUDA(cudaFuncSetAttribute(attn_fwd_kernel<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, FWD_SMEM));
    MB_CHECK_CUDA(cudaFuncSetAttribute(attn_fwd_kernel<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, FWD_SMEM));
    MB_CHECK_CUDA(cudaFuncSetAttribute(attn_fwd_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, FWD_SMEM));
    MB_CHECK_CUDA(cudaFuncSetAttribute(attn_fwd_kernel<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, FWD_SMEM));
    attr = true;
  }
  dim3 grid(ceil_div(a->S, AT_M), a->heads, a->B);
  const bool drop = a->dropout_p > 0.f;
  auto kern = a->valid ? (drop ? attn_fwd_kernel<true, true> : attn_fwd_kernel<true, false>)
                       : (drop ? attn_fwd_kernel<false, true> : attn_fwd_kernel<false, false>);
  MB_CHECK_CUDA(launch_pdl(kern, grid, dim3(FWD_THREADS), FWD_SMEM, stream, tq, tkv, p));
  MB_CHECK_LAUNCH();
  return MERLOT_OK;
}

// > 0 (S <= 512): the short-sequence kernels run and the workspace is left alone; its size and this count stay as they were so
// that callers sizing scratch from them keep working
extern "C" int merlot_attention_bwd_dq_parts(int S) {
  const int n_kv = ceil_div(S, AT_N);
  return n_kv <= MAX_DQ_PARTS ? n_kv : 0;
}

extern "C" size_t merlot_attention_bwd_workspace_bytes(int B, int S, int heads) {
  const int parts = merlot_attention_bwd_dq_parts(S);
  return (size_t)(parts > 0 ? parts : 1) * (size_t)B * S * heads * 64 * sizeof(float);
}

extern "C" int merlot_attention_bwd(const merlot_attn_t* a, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  int rc = check_common(a);
  if (rc) return rc;
  MB_REQUIRE(a->ctx && a->d_ctx && a->lse && a->dsum && a->dq_accum && a->dqkv, MERLOT_EINVAL,
             "attention_bwd: ctx, d_ctx, lse, dsum, dq_accum and dqkv are all required");
  MB_REQUIRE((a->ld_ctx % 8) == 0 && (a->ld_dqkv % 8) == 0 && (a->ld_dq % 4) == 0, MERLOT_ESHAPE,
             "attention_bwd: leading dimensions must keep 16-byte alignment");
  // before the first launch: a rejected call must leave dsum (and everything else) untouched
  MB_REQUIRE(a->S <= MAX_MASK_WORDS * 32 - AT_M, MERLOT_ESHAPE, "attention_bwd: sequence longer than %d keys", MAX_MASK_WORDS * 32 - AT_M);
  AttnDev p; fill_dev(a, &p);
  const int H = p.H;
  const long long tokens = (long long)a->B * a->S;
  CUtensorMap tq, tdo;
  rc = make_tmap_bf16_2d(&tq, a->qkv, (uint64_t)a->ld_qkv, (uint64_t)tokens, (uint64_t)a->ld_qkv, 64, BQ);
  if (rc) return rc;
  rc = make_tmap_bf16_2d(&tdo, a->d_ctx, (uint64_t)a->ld_ctx, (uint64_t)tokens, (uint64_t)a->ld_ctx, 64, BQ);
  if (rc) return rc;
  if (merlot_attention_bwd_dq_parts(a->S) > 0) {  // short sequences: the dQ kernel, then the dK/dV kernel; dq_accum is not used
    static_assert(SB_ROWS == BQ, "one 64-row tensor map serves both short-sequence kernels");
    static_assert(MAX_DQ_PARTS * AT_N <= SB_MASK_WORDS * 32, "the short-sequence kernels' validity masks hold 512 positions");
    CUtensorMap to;
    rc = make_tmap_bf16_2d(&to, a->ctx, (uint64_t)a->ld_ctx, (uint64_t)tokens, (uint64_t)a->ld_ctx, 64, SB_ROWS);
    if (rc) return rc;
    p.d_bias = a->d_bias_qkv;
    // [HAS_MASK][DROP]
    static void (*const kdq[2][2])(CUtensorMap, CUtensorMap, CUtensorMap, AttnDev) = {
        {attn_bwd_dq_kernel<false, false>, attn_bwd_dq_kernel<false, true>},
        {attn_bwd_dq_kernel<true, false>, attn_bwd_dq_kernel<true, true>}};
    static void (*const kdkv[2][2])(CUtensorMap, CUtensorMap, AttnDev) = {
        {attn_bwd_dkdv_kernel<false, false>, attn_bwd_dkdv_kernel<false, true>},
        {attn_bwd_dkdv_kernel<true, false>, attn_bwd_dkdv_kernel<true, true>}};
    static bool attr_short = false;
    if (!attr_short) {
      for (int i = 0; i < 4; ++i) {
        MB_CHECK_CUDA(cudaFuncSetAttribute(kdq[i >> 1][i & 1], cudaFuncAttributeMaxDynamicSharedMemorySize, DQ_SMEM));
        MB_CHECK_CUDA(cudaFuncSetAttribute(kdkv[i >> 1][i & 1], cudaFuncAttributeMaxDynamicSharedMemorySize, DKV_SMEM));
      }
      attr_short = true;
    }
    const int m = a->valid != nullptr, d = a->dropout_p > 0.f;
    dim3 grid(ceil_div(a->S, SB_ROWS), a->heads, a->B);
    MB_CHECK_CUDA(launch_pdl(kdq[m][d], grid, dim3(SB_THREADS), DQ_SMEM, stream, tq, tdo, to, p));
    MB_CHECK_LAUNCH();
    MB_CHECK_CUDA(launch_pdl(kdkv[m][d], grid, dim3(SB_THREADS), DKV_SMEM, stream, tq, tdo, p));
    MB_CHECK_LAUNCH();
    return MERLOT_OK;
  }
  {  // D = rowsum(dO * O)
    const long long threads = tokens * a->heads * 8;
    MB_CHECK_CUDA(launch_pdl(attn_dsum_kernel, dim3((unsigned)ceil_div_ll(threads, 256)), dim3(256), 0, stream,
                             reinterpret_cast<const bf16*>(a->ctx), reinterpret_cast<const bf16*>(a->d_ctx), a->ld_ctx, a->dsum,
                             a->B, a->S, a->heads));
    MB_CHECK_LAUNCH();
  }
  CUtensorMap tkv;
  rc = make_tmap_bf16_2d(&tkv, a->qkv, (uint64_t)a->ld_qkv, (uint64_t)tokens, (uint64_t)a->ld_qkv, 64, AT_N);
  if (rc) return rc;
  // [HAS_MASK][DROP]
  static void (*const kerns[2][2])(CUtensorMap, CUtensorMap, CUtensorMap, AttnDev) = {
      {attn_bwd_kernel<false, false>, attn_bwd_kernel<false, true>},
      {attn_bwd_kernel<true, false>, attn_bwd_kernel<true, true>}};
  static bool attr = false;
  if (!attr) {
    for (int i = 0; i < 4; ++i)
      MB_CHECK_CUDA(cudaFuncSetAttribute(kerns[i >> 1][i & 1], cudaFuncAttributeMaxDynamicSharedMemorySize, BWD_SMEM));
    attr = true;
  }
  dim3 grid(ceil_div(a->S, AT_N), a->heads, a->B);
  MB_CHECK_CUDA(launch_pdl(kerns[a->valid != nullptr][a->dropout_p > 0.f], grid, dim3(BWD_THREADS), BWD_SMEM, stream, tkv, tq, tdo, p));
  MB_CHECK_LAUNCH();
  {
    long long slabs = ceil_div_ll(tokens, 64);
    if (slabs > 128) slabs = 128;
    MB_CHECK_CUDA(launch_pdl(attn_dqkv_finish_kernel, dim3(ceil_div(3 * H, 256), (unsigned)slabs), dim3(256), 0, stream, a->dq_accum,
                             a->ld_dq, p.dqkv, a->ld_dqkv, tokens, H, a->d_bias_qkv, a->scale));
    MB_CHECK_LAUNCH();
  }
  return MERLOT_OK;
}

// attention_log (model/modeling.py:186-203): 4 normalised block sums from the split column sums.
//   c_viz[b,k] / c_lang[b,k] = sum over (layers, valid queries in the viz / lang piece) of head-mean probabilities
//   out = {lang2lang, lang2viz, viz2lang, viz2viz}  (names are `from`2`to`: keys are `from`, queries are `to`), sum = 1
__global__ void attn_log_blocks_kernel(const float* __restrict__ c_viz, const float* __restrict__ c_lang, const uint8_t* __restrict__ valid,
                                       int B, int S, int P, float* __restrict__ out) {
  __shared__ float red[4][256];
  float a[4] = {0.f, 0.f, 0.f, 0.f};  // [to_viz_from_viz, to_viz_from_lang, to_lang_from_viz, to_lang_from_lang]
  for (int i = threadIdx.x; i < B * S; i += 256) {
    const int k = i % S;
    const float vk = valid[i] ? 1.f : 0.f;
    const int from_lang = k >= P;
    a[0 + from_lang] += c_viz[i] * vk;
    a[2 + from_lang] += c_lang[i] * vk;
  }
  for (int j = 0; j < 4; ++j) red[j][threadIdx.x] = a[j];
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o)
      for (int j = 0; j < 4; ++j) red[j][threadIdx.x] += red[j][threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const float tot = red[0][0] + red[1][0] + red[2][0] + red[3][0];
    out[0] = red[3][0] / tot;  // lang2lang : keys lang, queries lang
    out[1] = red[1][0] / tot;  // lang2viz  : keys lang, queries viz
    out[2] = red[2][0] / tot;  // viz2lang  : keys viz,  queries lang
    out[3] = red[0][0] / tot;  // viz2viz
  }
}

extern "C" int merlot_attention_log_blocks(const float* c_viz, const float* c_lang, const void* valid, int B, int S, int P, float* out4,
                                           void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  MB_REQUIRE(c_viz && c_lang && valid && out4, MERLOT_EINVAL, "attention_log_blocks: null pointer");
  attn_log_blocks_kernel<<<1, 256, 0, stream>>>(c_viz, c_lang, reinterpret_cast<const uint8_t*>(valid), B, S, P, out4);
  MB_CHECK_LAUNCH();
  return MERLOT_OK;
}

extern "C" int merlot_attention_colsum(const merlot_attn_t* a, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  int rc = check_common(a);
  if (rc) return rc;
  MB_REQUIRE(a->lse && a->colsum, MERLOT_EINVAL, "attention_colsum: lse and colsum are required");
  AttnDev p; fill_dev(a, &p);
  CUtensorMap tk, tq;
  rc = make_tmap_bf16_2d(&tk, a->qkv, (uint64_t)a->ld_qkv, (uint64_t)a->B * a->S, (uint64_t)a->ld_qkv, 64, AT_N);
  if (rc) return rc;
  rc = make_tmap_bf16_2d(&tq, a->qkv, (uint64_t)a->ld_qkv, (uint64_t)a->B * a->S, (uint64_t)a->ld_qkv, 64, BQ);
  if (rc) return rc;
  MB_REQUIRE(a->S <= MAX_MASK_WORDS * 32 - AT_M, MERLOT_ESHAPE, "attention_colsum: sequence longer than %d keys", MAX_MASK_WORDS * 32 - AT_M);
  static bool attr = false;
  if (!attr) {
    MB_CHECK_CUDA(cudaFuncSetAttribute(attn_colsum_kernel<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, CS_SMEM));
    MB_CHECK_CUDA(cudaFuncSetAttribute(attn_colsum_kernel<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, CS_SMEM));
    MB_CHECK_CUDA(cudaFuncSetAttribute(attn_colsum_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, CS_SMEM));
    MB_CHECK_CUDA(cudaFuncSetAttribute(attn_colsum_kernel<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, CS_SMEM));
    attr = true;
  }
  dim3 grid(ceil_div(a->S, AT_N), a->heads, a->B);
  const bool drop = a->dropout_p > 0.f;
  auto kern = a->valid ? (drop ? attn_colsum_kernel<true, true> : attn_colsum_kernel<true, false>)
                       : (drop ? attn_colsum_kernel<false, true> : attn_colsum_kernel<false, false>);
  MB_CHECK_CUDA(launch_pdl(kern, grid, dim3(CS_THREADS), CS_SMEM, stream, tk, tq, p));
  MB_CHECK_LAUNCH();
  return MERLOT_OK;
}
