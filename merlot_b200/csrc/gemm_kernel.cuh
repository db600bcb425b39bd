// K1 kernel template and its launch dispatch; instantiated per tile width in gemm_bn{128,192,256}.cu so the three widths
// compile in parallel (4 operand-major combinations each).
#pragma once
#include "gemm_common.cuh"

namespace mb {

// Fused epilogue of one warp's [16 rows][64 columns] fp32 slot (float4 units XOR-swizzled by row): lane l handles the 8-column
// groups l, l + 32, l + 64, l + 96 (row = group / 8), so 8 lanes cover one row's 256 contiguous bytes.  Inlined: a call would
// have to save every live accumulator register around it.
static __device__ __forceinline__ void gemm_epilogue_slot(const GemmDev& p, const float* slot, int row0, int col0, int lane) {
#pragma unroll 1
  for (int it = 0; it < 4; ++it) {
    const int item = it * 32 + lane;
    const int rr = item >> 3, g = item & 7;
    const int row = row0 + rr, col = col0 + g * 8;
    if (row >= p.M || col >= p.N) continue;
    const float4 lo = *reinterpret_cast<const float4*>(slot + rr * 64 + (((2 * g) ^ rr) << 2));
    const float4 hi = *reinterpret_cast<const float4*>(slot + rr * 64 + (((2 * g + 1) ^ rr) << 2));
    float v[8] = {lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z, hi.w}, pre[8];
    epi_math8(p, row, col, true, v, pre);
    epi_store_direct(p, row, col, v, pre);
  }
}

template <int BN>
__device__ __forceinline__ void wgmma_tile(float (&acc)[BN / 2], uint64_t da, uint64_t db, uint32_t scale_d, bool a_mn, bool b_mn);

#define MB_WGMMA_TILE(N)                                                                                                      \
  template <>                                                                                                                 \
  __device__ __forceinline__ void wgmma_tile<N>(float (&acc)[N / 2], uint64_t da, uint64_t db, uint32_t sd, bool a_mn, bool b_mn) { \
    if (a_mn) {                                                                                                               \
      if (b_mn) wgmma_m64n##N##_ss<1, 1>(acc, da, db, sd); else wgmma_m64n##N##_ss<1, 0>(acc, da, db, sd);                    \
    } else {                                                                                                                  \
      if (b_mn) wgmma_m64n##N##_ss<0, 1>(acc, da, db, sd); else wgmma_m64n##N##_ss<0, 0>(acc, da, db, sd);                    \
    }                                                                                                                         \
  }
MB_WGMMA_TILE(128)
MB_WGMMA_TILE(192)
MB_WGMMA_TILE(256)
#undef MB_WGMMA_TILE

// Persistent, warp-specialised bf16 GEMM (static tile schedule, split-K for the wgrad orientation):
//   warp 0 (one elected lane): TMA producer -- A/B tiles -> 128B-swizzled smem ring of STAGES stages; it runs ahead across
//                              tiles, so the loads of tile i+1 overlap the epilogue of tile i;
//   warpgroups 1, 2:           rows [0, 64) / [64, 128) of the tile: m64 x BN x 16 wgmma with fp32 accumulators in registers,
//                              one k-block in flight behind the one being issued, then the fused epilogue.
template <int BN, bool A_MN, bool B_MN>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_bf16_kernel(const __grid_constant__ CUtensorMap tma_a, const __grid_constant__ CUtensorMap tma_b, const GemmDev p) {
  using Cfg = GemmCfg<BN>;
  constexpr int STAGES = Cfg::STAGES;
  extern __shared__ uint8_t smem_raw[];
  // 128B swizzle atoms need 1024-byte alignment
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + STAGES * Cfg::A_BYTES;
  float* staging = reinterpret_cast<float*>(smem + STAGES * Cfg::STAGE_BYTES);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + STAGES * Cfg::STAGE_BYTES + STAGING_BYTES);
  uint64_t* empty_bar = full_bar + STAGES;

  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);  // provably warp-uniform
  const int lane = threadIdx.x & 31;
  pdl_launch_dependents();

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tma_a);
    tma_prefetch_desc(&tma_b);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 2);  // one arrival per consumer warpgroup
    }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();  // everything above overlapped the previous kernel's tail

  const int num_tiles = p.m_blocks * p.n_blocks * p.splits;

  if (warp < 4) {
    // ===================== TMA producer =====================
    // the producer warpgroup hands registers to the consumers (40 + 2 x 232 per thread x 128 <= 64 K)
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;\n" ::: "memory");
    if (warp == 0 && elect_one()) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int split = tile % p.splits;
        const int mn = tile / p.splits;
        const int n_blk = mn % p.n_blocks;
        const int m_blk = mn / p.n_blocks;
        const int kb0 = split * p.kb_per_split;
        const int kb1 = min(p.num_kb, kb0 + p.kb_per_split);
        for (int kb = kb0; kb < kb1; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          mbar_arrive_expect_tx(&full_bar[stage], Cfg::STAGE_BYTES);
          uint8_t* sa = smem_a + stage * Cfg::A_BYTES;
          uint8_t* sb = smem_b + stage * Cfg::B_BYTES;
          if (A_MN) {
#pragma unroll
            for (int c = 0; c < BLOCK_M / 64; ++c)
              tma_load_2d(sa + c * (BLOCK_K * 128), &tma_a, &full_bar[stage], m_blk * BLOCK_M + c * 64, kb * BLOCK_K);
          } else {
            tma_load_2d(sa, &tma_a, &full_bar[stage], kb * BLOCK_K, m_blk * BLOCK_M);
          }
          if (B_MN) {
#pragma unroll
            for (int c = 0; c < BN / 64; ++c)
              tma_load_2d(sb + c * (BLOCK_K * 128), &tma_b, &full_bar[stage], n_blk * BN + c * 64, kb * BLOCK_K);
          } else {
            tma_load_2d(sb, &tma_b, &full_bar[stage], kb * BLOCK_K, n_blk * BN);
          }
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // ===================== consumer warpgroups =====================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;\n" ::: "memory");
    const int wg = (warp - 4) >> 2;  // rows [64 wg, 64 wg + 64) of the tile
    const int wq = warp & 3;         // 16-row slice of this warp inside the warpgroup's 64 rows
    const bool wg_leader = (threadIdx.x & 127) == 0;
    float* slot = staging + (warp - 4) * 1024;
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int split = tile % p.splits;
      const int mn = tile / p.splits;
      const int n_blk = mn % p.n_blocks;
      const int m_blk = mn / p.n_blocks;
      const int kb0 = split * p.kb_per_split;
      const int kb1 = min(p.num_kb, kb0 + p.kb_per_split);
      int prev = -1;
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t a_addr = smem_u32(smem_a + stage * Cfg::A_BYTES) + (uint32_t)wg * (A_MN ? BLOCK_K * 128 : 64 * 128);
        const uint32_t b_addr = smem_u32(smem_b + stage * Cfg::B_BYTES);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BLOCK_K / 16; ++k) {
          const uint64_t da = A_MN ? desc_mnmajor(a_addr, k, BLOCK_K * 128) : desc_kmajor(a_addr, k);
          const uint64_t db = B_MN ? desc_mnmajor(b_addr, k, BLOCK_K * 128) : desc_kmajor(b_addr, k);
          wgmma_tile<BN>(acc, da, db, (kb > kb0 || k > 0) ? 1u : 0u, A_MN, B_MN);
        }
        wgmma_commit();
        wgmma_wait<1>();  // the k-block before this one has been read: its stage goes back to the producer
        if (prev >= 0 && wg_leader) mbar_arrive(&empty_bar[prev]);
        prev = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      reg_fence(acc);
      if (prev >= 0 && wg_leader) mbar_arrive(&empty_bar[prev]);
      // ---- epilogue: 64-column chunks through the warp's slot ----
      // A run-time loop over the chunks, so the fused epilogue (every flag's path) is in the kernel once rather than once
      // per chunk: unrolled, it made the kernel too large for the instruction cache and the fetch misses slowed the whole
      // tile loop.  Only the register -> slot copy is unrolled per chunk (accumulator indices must be compile-time).
      const int row0 = m_blk * BLOCK_M + wg * 64 + wq * 16;
      const int r = lane >> 2;
#pragma unroll 1
      for (int c = 0; c < BN / 64; ++c) {
        __syncwarp();
#pragma unroll
        for (int cc = 0; cc < BN / 64; ++cc) {
          if (cc != c) continue;
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) {
            const int j = cc * 8 + jj;
            const int unit = jj * 2 + ((lane & 3) >> 1), within = (lane & 1) * 2;
            *reinterpret_cast<float2*>(slot + r * 64 + ((unit ^ r) << 2) + within) = make_float2(acc[4 * j], acc[4 * j + 1]);
            *reinterpret_cast<float2*>(slot + (r + 8) * 64 + ((unit ^ (r + 8)) << 2) + within) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
          }
        }
        __syncwarp();
        if (n_blk * BN + c * 64 < p.N) gemm_epilogue_slot(p, slot, row0, n_blk * BN + c * 64, lane);
      }
    }
  }
}

template <int BN, bool A_MN, bool B_MN>
static int launch_gemm_inst(const CUtensorMap& ta, const CUtensorMap& tb, const GemmDev& p, int grid, cudaStream_t stream) {
  using Cfg = GemmCfg<BN>;
  auto kern = gemm_bf16_kernel<BN, A_MN, B_MN>;
  static bool attr_set = false;  // per instantiation
  if (!attr_set) {
    MB_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_TOTAL));
    attr_set = true;
  }
  void* tok = gemm_prof_before(2.0 * (double)p.M * (double)p.N * (double)p.K, stream);
  MB_CHECK_CUDA(launch_pdl(kern, dim3(grid), dim3(GEMM_THREADS), Cfg::SMEM_TOTAL, stream, ta, tb, p));
  MB_CHECK_LAUNCH();
  gemm_prof_after(tok, stream);
  return MERLOT_OK;
}

template <int BN>
int launch_gemm_bn(bool a_mn, bool b_mn, const CUtensorMap& ta, const CUtensorMap& tb, const GemmDev& p, int grid, cudaStream_t stream) {
  if (a_mn && b_mn) return launch_gemm_inst<BN, true, true>(ta, tb, p, grid, stream);
  if (!a_mn && b_mn) return launch_gemm_inst<BN, false, true>(ta, tb, p, grid, stream);
  if (!a_mn && !b_mn) return launch_gemm_inst<BN, false, false>(ta, tb, p, grid, stream);
  return launch_gemm_inst<BN, true, false>(ta, tb, p, grid, stream);
}

}  // namespace mb
