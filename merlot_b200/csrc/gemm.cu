// K1: persistent, warp-specialised bf16 GEMM for sm_90a (kernel in gemm_kernel.cuh).
//   warp 0           : TMA producer (one elected lane) -- A/B tiles -> 128B-swizzled smem ring (full/empty mbarriers)
//   warpgroups 1, 2  : wgmma 64 x BN x 16 each (fp32 accumulators in registers) -> fused epilogue -> TMA stores (fast kinds)
//                      or vectorised global stores (generic epilogue)
// Host side: argument checks, tile width, split-K, epilogue kind, tensor maps.
//
// Replaces the reference's tf.layers.dense / tf.matmul call sites listed in include/merlot_b200.h (K1).
#include "gemm_common.cuh"

#include <stdlib.h>

#include <vector>

namespace mb {

// Optional per-launch timing (bench.py roofline): CUDA events on the launching stream around every GEMM launch.
struct ProfRec { cudaEvent_t e0, e1; double flops; };
static bool g_prof_on = false;
static std::vector<ProfRec> g_prof;

void* gemm_prof_before(double flops, cudaStream_t stream) {
  if (!g_prof_on) return nullptr;
  ProfRec* rec = new ProfRec;
  rec->flops = flops;
  cudaEventCreate(&rec->e0);
  cudaEventCreate(&rec->e1);
  cudaEventRecord(rec->e0, stream);
  return rec;
}
void gemm_prof_after(void* tok, cudaStream_t stream) {
  if (!tok) return;
  ProfRec* rec = reinterpret_cast<ProfRec*>(tok);
  cudaEventRecord(rec->e1, stream);
  g_prof.push_back(*rec);
  delete rec;
}

}  // namespace mb

namespace mb {
template <int BN>
int launch_gemm_bn(bool a_mn, bool b_mn, int kind, const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& to,
                   const CUtensorMap& to2, const GemmDev& p, int grid, cudaStream_t stream);  // gemm_bn{128,192,256}.cu

// The fast epilogue (EpiKind, gemm_common.cuh) for this launch, or EPI_GENERIC.  It needs alpha = 1, whole 8-column groups
// (N % 8 == 0), a bias that float2 loads can read, and outputs TMA can address (16-byte base, 16-byte row pitch).  The
// flag word seen here has DROPOUT cleared when p = 0.
static int epilogue_kind(const merlot_gemm_t* g, uint32_t flags, int bn) {
  if ((flags & (MERLOT_GEMM_GENERIC_EPILOGUE | MERLOT_GEMM_MUL_DGELU)) || g->alpha != 1.f || (g->N % 8) != 0 ||
      ((uintptr_t)g->bias % 8) != 0)
    return EPI_GENERIC;
  if (flags & MERLOT_GEMM_OUT_F32) {
    const bool red_only = (flags & MERLOT_GEMM_ATOMIC) && !(flags & ~(MERLOT_GEMM_OUT_F32 | MERLOT_GEMM_ATOMIC)) && !g->bias &&
                          !g->resid;
    return (red_only && bn == 256 && ((uintptr_t)g->out % 16) == 0 && (g->ld_out % 4) == 0) ? EPI_RED_F32 : EPI_GENERIC;
  }
  if (flags & MERLOT_GEMM_GELU)
    return (g->out2 && !g->resid && !(flags & (MERLOT_GEMM_DROPOUT | MERLOT_GEMM_MUL_AUX))) ? EPI_GELU2 : EPI_GENERIC;
  // Plain, bias, residual and dropout bf16 outputs stay generic: through per-warp TMA stores they measured slower (up to
  // 1.7x on the joint encoder's N = 768 GEMMs), with no side input whose latency the fast path would hide.
  return (flags == MERLOT_GEMM_MUL_AUX && !g->bias && !g->resid) ? EPI_MUL_AUX : EPI_GENERIC;
}
}

using namespace mb;

extern "C" int merlot_gemm_bf16(const merlot_gemm_t* g, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  MB_REQUIRE(g != nullptr, MERLOT_EINVAL, "gemm: null descriptor");
  MB_REQUIRE(g->a && g->b && g->out, MERLOT_EINVAL, "gemm: null operand pointer");
  MB_REQUIRE(g->M > 0 && g->N > 0 && g->K > 0, MERLOT_ESHAPE, "gemm: non-positive dims M=%d N=%d K=%d", g->M, g->N,
             g->K);
  MB_REQUIRE((g->lda % 8) == 0 && (g->ldb % 8) == 0, MERLOT_ESHAPE,
             "gemm: lda/ldb must be multiples of 8 bf16 elements for TMA (lda=%d ldb=%d)", g->lda, g->ldb);
  MB_REQUIRE(((uintptr_t)g->a % 16) == 0 && ((uintptr_t)g->b % 16) == 0, MERLOT_ESHAPE,
             "gemm: operand base pointers must be 16-byte aligned");
  MB_REQUIRE(g->lda >= (g->a_mn_major ? g->M : g->K) && g->ldb >= (g->b_mn_major ? g->N : g->K), MERLOT_ESHAPE,
             "gemm: leading dimension smaller than the row length");
  const bool out_f32 = g->flags & MERLOT_GEMM_OUT_F32;
  MB_REQUIRE(!(g->flags & MERLOT_GEMM_ATOMIC) || out_f32, MERLOT_EINVAL, "gemm: ATOMIC requires OUT_F32");
  MB_REQUIRE(!(g->flags & (MERLOT_GEMM_MUL_DGELU | MERLOT_GEMM_MUL_AUX)) || g->aux, MERLOT_EINVAL, "gemm: MUL_DGELU / MUL_AUX require aux");
  MB_REQUIRE(!((g->flags & MERLOT_GEMM_MUL_DGELU) && (g->flags & MERLOT_GEMM_MUL_AUX)), MERLOT_EINVAL, "gemm: MUL_DGELU and MUL_AUX are exclusive");
  MB_REQUIRE(!(g->flags & MERLOT_GEMM_GELU_GRAD_OUT) || ((g->flags & MERLOT_GEMM_GELU) && g->out2), MERLOT_EINVAL,
             "gemm: GELU_GRAD_OUT needs GELU and out2");
  MB_REQUIRE(g->ld_out >= g->N, MERLOT_ESHAPE, "gemm: ld_out < N");
  if (!out_f32)
    MB_REQUIRE((g->ld_out % 8) == 0 && ((uintptr_t)g->out % 16) == 0, MERLOT_ESHAPE,
               "gemm: bf16 output needs ld_out %% 8 == 0 and a 16-byte aligned base");
  if (g->resid) MB_REQUIRE((g->ld_resid % 8) == 0 && ((uintptr_t)g->resid % 16) == 0, MERLOT_ESHAPE, "gemm: resid needs ld_resid %% 8 == 0 and a 16-byte aligned base");
  if (g->aux) MB_REQUIRE((g->ld_aux % 8) == 0 && ((uintptr_t)g->aux % 16) == 0, MERLOT_ESHAPE, "gemm: aux needs ld_aux %% 8 == 0 and a 16-byte aligned base");
  if (g->out2) MB_REQUIRE((g->ld_out2 % 8) == 0, MERLOT_ESHAPE, "gemm: ld_out2 %% 8 != 0");
  if (g->flags & MERLOT_GEMM_DROPOUT)
    MB_REQUIRE((g->N % 8) == 0 && g->dropout_p >= 0.f && g->dropout_p < 1.f, MERLOT_ESHAPE,
               "gemm: dropout needs N %% 8 == 0 and 0 <= p < 1");

  GemmDev p;
  memset(&p, 0, sizeof(p));
  p.M = g->M; p.N = g->N; p.K = g->K;
  p.out = g->out; p.ld_out = g->ld_out; p.out2 = g->out2; p.ld_out2 = g->ld_out2;
  p.bias = g->bias;
  p.resid = reinterpret_cast<const bf16*>(g->resid); p.ld_resid = g->ld_resid;
  p.aux = reinterpret_cast<const bf16*>(g->aux); p.ld_aux = g->ld_aux;
  p.alpha = g->alpha;
  p.flags = g->flags;
  if ((g->flags & MERLOT_GEMM_DROPOUT) && g->dropout_p > 0.f) {
    p.drop_thresh16 = (uint32_t)(g->dropout_p * 65536.0f + 0.5f);
    p.drop_scale = 1.0f / (1.0f - g->dropout_p);
    p.seed = g->dropout_seed;
    p.site = g->dropout_site;
  } else {
    p.flags &= ~MERLOT_GEMM_DROPOUT;
  }

  const int sms = num_sms();
  p.m_blocks = ceil_div(g->M, BLOCK_M);
  p.num_kb = ceil_div(g->K, BLOCK_K);
  // ---- tile width: minimise wave-quantisation loss; BN=256 halves per-FLOP smem traffic so it wins ties ----
  int bn = g->block_n;
  if (bn == 0 && (g->flags & MERLOT_GEMM_ATOMIC)) bn = 256;  // wgrad: split-K fills the machine, wide tiles halve smem traffic
  if (bn == 0) {
    double best = -1;
    for (int cand : {256, 192, 128}) {
      long long tiles = (long long)p.m_blocks * ceil_div(g->N, cand);
      long long waves = ceil_div_ll(tiles, sms);
      double useful = (double)g->N / (double)(ceil_div(g->N, cand) * cand);
      double eff = (double)tiles / (double)(waves * sms) * useful * (cand == 256 ? 1.0 : (cand == 192 ? 0.97 : 0.80));
      if (eff > best + 1e-9) { best = eff; bn = cand; }
    }
  }
  MB_REQUIRE(bn == 128 || bn == 192 || bn == 256, MERLOT_EINVAL, "gemm: block_n must be 0, 128, 192 or 256 (got %d)", bn);
  p.n_blocks = ceil_div(g->N, bn);
  // ---- split-K (wgrad): fill the machine when the MN tile count is small ----
  int splits = g->splits;
  const int mn_tiles = p.m_blocks * p.n_blocks;
  if (splits <= 0) {
    splits = 1;
    if ((g->flags & MERLOT_GEMM_ATOMIC) && mn_tiles < sms) {
      splits = sms / mn_tiles;
      int max_by_k = p.num_kb / 4 > 0 ? p.num_kb / 4 : 1;  // keep >= 4 k-blocks per split
      if (splits > max_by_k) splits = max_by_k;
      if (splits < 1) splits = 1;
    }
  }
  MB_REQUIRE(splits == 1 || (g->flags & MERLOT_GEMM_ATOMIC), MERLOT_EINVAL, "gemm: splits>1 requires ATOMIC");
  if (splits > p.num_kb) splits = p.num_kb;
  p.kb_per_split = ceil_div(p.num_kb, splits);
  p.splits = ceil_div(p.num_kb, p.kb_per_split);  // no empty splits

  CUtensorMap ta, tb;
  int rc;
  if (g->a_mn_major)
    rc = make_tmap_bf16_2d(&ta, g->a, (uint64_t)g->M, (uint64_t)g->K, (uint64_t)g->lda, 64, BLOCK_K);
  else
    rc = make_tmap_bf16_2d(&ta, g->a, (uint64_t)g->K, (uint64_t)g->M, (uint64_t)g->lda, BLOCK_K, BLOCK_M);
  if (rc) return rc;
  if (g->b_mn_major)
    rc = make_tmap_bf16_2d(&tb, g->b, (uint64_t)g->N, (uint64_t)g->K, (uint64_t)g->ldb, 64, BLOCK_K);
  else
    rc = make_tmap_bf16_2d(&tb, g->b, (uint64_t)g->K, (uint64_t)g->N, (uint64_t)g->ldb, BLOCK_K, (uint32_t)bn);
  if (rc) return rc;

  const long long tiles = (long long)mn_tiles * p.splits;
  const int grid = (int)(tiles < sms ? tiles : sms);
  if ((g->flags & MERLOT_GEMM_GELU) && g->out2 && !out_f32)
    MB_REQUIRE(((uintptr_t)g->out2 % 16) == 0, MERLOT_ESHAPE, "gemm: out2 must be 16-byte aligned");

  // fast epilogue: output tensor maps, one warp's [16 rows][128 B] sub-tile per box; TMA clips at M and N
  const int kind = epilogue_kind(g, p.flags, bn);
  CUtensorMap to, to2;
  memset(&to, 0, sizeof(to));
  memset(&to2, 0, sizeof(to2));
  if (kind == EPI_RED_F32) {
    rc = make_tmap_f32_2d(&to, g->out, (uint64_t)g->N, (uint64_t)g->M, (uint64_t)g->ld_out, 32, 16);
    if (rc) return rc;
  } else if (kind != EPI_GENERIC) {
    rc = make_tmap_bf16_2d(&to, g->out, (uint64_t)g->N, (uint64_t)g->M, (uint64_t)g->ld_out, 64, 16);
    if (rc) return rc;
    if (kind == EPI_GELU2) {
      rc = make_tmap_bf16_2d(&to2, g->out2, (uint64_t)g->N, (uint64_t)g->M, (uint64_t)g->ld_out2, 64, 16);
      if (rc) return rc;
    }
  }
  const bool a_mn = g->a_mn_major != 0, b_mn = g->b_mn_major != 0;
  if (bn == 256) return launch_gemm_bn<256>(a_mn, b_mn, kind, ta, tb, to, to2, p, grid, stream);
  if (bn == 192) return launch_gemm_bn<192>(a_mn, b_mn, kind, ta, tb, to, to2, p, grid, stream);
  return launch_gemm_bn<128>(a_mn, b_mn, kind, ta, tb, to, to2, p, grid, stream);
}

extern "C" void merlot_gemm_profile_begin(void) {
  for (auto& r : g_prof) { cudaEventDestroy(r.e0); cudaEventDestroy(r.e1); }
  g_prof.clear();
  g_prof_on = true;
}

extern "C" int merlot_gemm_profile_end(double* total_ms, double* total_flops, long long* launches) {
  g_prof_on = false;
  MB_CHECK_CUDA(cudaDeviceSynchronize());
  double ms = 0, fl = 0;
  for (auto& r : g_prof) {
    float t = 0.f;
    MB_CHECK_CUDA(cudaEventElapsedTime(&t, r.e0, r.e1));
    ms += t; fl += r.flops;
    cudaEventDestroy(r.e0); cudaEventDestroy(r.e1);
  }
  if (total_ms) *total_ms = ms;
  if (total_flops) *total_flops = fl;
  if (launches) *launches = (long long)g_prof.size();
  g_prof.clear();
  return MERLOT_OK;
}
