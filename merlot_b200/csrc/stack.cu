// Native driver of one pre-LN transformer stack (utils/transformer.py:171-247): forward and hand-written backward,
// enqueuing the K1/K2/K3/K5 kernels of this library on one stream.  The reference builds this loop in Python/TF and lets
// tf.gradients derive the backward graph (utils/optimization.py:176); here both directions are explicit.
//
// Per layer (residual stream h is bf16, statistics fp32):
//   x1 = LN(h); qkv = x1 Wqkv + b; ctx = attn(qkv); hmid = h + drop(ctx Wo + bo);
//   x2 = LN(hmid); pre = x2 W1 + b1; act = gelu(pre); hout = hmid + drop(act W2 + b2)
// and y = LN_final(h_last).  Weights are bf16 copies in the reference's [in,out] layout: the forward GEMM reads them as
// an MN-major B operand, dgrad reads the same buffer as a K-major B operand, wgrad reads both activations MN-major and
// red.adds fp32 into the flat gradient arena (so the shared `encoder` weights accumulate both of their passes).
#include "host_common.h"

#include <map>
#include <mutex>

namespace mb {

// Weight-gradient GEMMs run on a companion stream of the stream the backward pass is enqueued on: a persistent K1 launch
// leaves the SMs of its last partial wave idle (1.4-5.4 waves per GEMM at these shapes), and wgrad(W) and dgrad(x) of a layer
// are independent, so the other stream's CTAs fill those tails.  Events order each wgrad behind the kernel that produces its
// dy and hold back the kernel that overwrites that dy until the wgrad has read it.
struct WgradLane {
  cudaStream_t stream = nullptr;
  cudaEvent_t ready[4] = {nullptr, nullptr, nullptr, nullptr};  // recorded on the main stream: dy of wgrad i is final
  cudaEvent_t done[4] = {nullptr, nullptr, nullptr, nullptr};   // recorded on the lane: wgrad i has read its operands
};
static WgradLane* wgrad_lane(cudaStream_t main) {
  static std::map<cudaStream_t, WgradLane> lanes;
  static std::mutex mu;
  static const bool off = [] { const char* e = getenv("MERLOT_WGRAD_STREAM"); return e && e[0] == '0'; }();
  if (off) return nullptr;
  const char* e = getenv("MERLOT_NO_SIDE_STREAM");  // single-stream diagnostics (bench.py's per-launch event timing)
  if (e && e[0] == '1') return nullptr;
  std::lock_guard<std::mutex> lock(mu);
  WgradLane& w = lanes[main];
  if (w.stream == nullptr) {
    if (cudaStreamCreateWithFlags(&w.stream, cudaStreamNonBlocking) != cudaSuccess) { w.stream = nullptr; return nullptr; }
    for (int i = 0; i < 4; ++i) {
      cudaEventCreateWithFlags(&w.ready[i], cudaEventDisableTiming);
      cudaEventCreateWithFlags(&w.done[i], cudaEventDisableTiming);
    }
  }
  return &w;
}

static inline size_t align_up(size_t x, size_t a = 256) { return (x + a - 1) / a * a; }

struct LayerAct {
  char *x1, *qkv, *ctx, *hmid, *x2, *pre, *act, *hout;
  float *lse, *mean1, *rstd1, *mean2, *rstd2;
};

static size_t layer_act_bytes(const merlot_stack_t* s) {
  const size_t M = (size_t)s->B * s->S, H = s->H, I = s->I;
  return align_up(M * H * 2) * 5 + align_up(M * 3 * H * 2) + align_up(M * I * 2) * 2 +
         align_up((size_t)s->B * s->heads * s->S * 4) + align_up(M * 4) * 4;
}

static LayerAct carve(const merlot_stack_t* s, char* base) {
  const size_t M = (size_t)s->B * s->S, H = s->H, I = s->I;
  LayerAct a;
  char* p = base;
  auto take = [&](size_t n) { char* r = p; p += align_up(n); return r; };
  a.x1 = take(M * H * 2); a.qkv = take(M * 3 * H * 2); a.ctx = take(M * H * 2); a.hmid = take(M * H * 2);
  a.x2 = take(M * H * 2); a.pre = take(M * I * 2); a.act = take(M * I * 2); a.hout = take(M * H * 2);
  a.lse = (float*)take((size_t)s->B * s->heads * s->S * 4);
  a.mean1 = (float*)take(M * 4); a.rstd1 = (float*)take(M * 4); a.mean2 = (float*)take(M * 4); a.rstd2 = (float*)take(M * 4);
  return a;
}

static int check_stack(const merlot_stack_t* s) {
  MB_REQUIRE(s != nullptr, MERLOT_EINVAL, "stack: null descriptor");
  MB_REQUIRE(s->B > 0 && s->S > 0 && s->layers > 0, MERLOT_ESHAPE, "stack: bad dims B=%d S=%d layers=%d", s->B, s->S, s->layers);
  MB_REQUIRE(s->H == s->heads * 64, MERLOT_ESHAPE,
             "stack: hidden_size %d != num_attention_heads %d * 64 (utils/transformer.py:16-19 raises ValueError on the same mismatch)",
             s->H, s->heads);
  MB_REQUIRE(s->H % 8 == 0 && s->I % 8 == 0 && s->H <= 1024, MERLOT_ESHAPE, "stack: H, I must be multiples of 8 and H <= 1024");
  MB_REQUIRE(s->layer_params && s->h_in && s->act_arena && s->final_gamma && s->final_beta, MERLOT_EINVAL, "stack: null pointer");
  MB_REQUIRE(s->attention_dropout_p >= 0.f && s->attention_dropout_p < 1.f, MERLOT_EINVAL,
             "stack: attention_probs_dropout_prob must lie in [0, 1) (got %g)", (double)s->attention_dropout_p);
  return MERLOT_OK;
}

static int ln_fwd(const void* x, void* y, const float* g, const float* b, float* mean, float* rstd, long long rows, int H,
                  cudaStream_t st) {
  merlot_ln_t d;
  memset(&d, 0, sizeof(d));
  d.x = x; d.ld_x = H; d.y = y; d.ld_y = H; d.gamma = g; d.beta = b; d.mean = mean; d.rstd = rstd; d.rows = rows; d.H = H;
  d.eps = 1e-5f;
  return merlot_layernorm_fwd(&d, st);
}

static merlot_gemm_t gemm_base(int M, int N, int K) {
  merlot_gemm_t g;
  memset(&g, 0, sizeof(g));
  g.M = M; g.N = N; g.K = K; g.alpha = 1.f;
  return g;
}

// y[M,N] = x[M,K] @ W[K,N] + bias (+ epilogue)
static int linear_fwd(const void* x, int K, const void* W, int N, const float* bias, int M, merlot_gemm_t extra, cudaStream_t st) {
  merlot_gemm_t g = extra;
  g.M = M; g.N = N; g.K = K;
  g.a = x; g.lda = K; g.a_mn_major = 0;
  g.b = W; g.ldb = N; g.b_mn_major = 1;
  g.bias = bias;
  return merlot_gemm_bf16(&g, st);
}
// dW[K,N] += x[M,K]^T @ dy[M,N]
static int linear_wgrad(const void* x, int K, const void* dy, int N, float* dW, int M, cudaStream_t st) {
  merlot_gemm_t g = gemm_base(K, N, M);
  g.a = x; g.lda = K; g.a_mn_major = 1;
  g.b = dy; g.ldb = N; g.b_mn_major = 1;
  g.out = dW; g.ld_out = N;
  g.flags = MERLOT_GEMM_OUT_F32 | MERLOT_GEMM_ATOMIC;
  return merlot_gemm_bf16(&g, st);
}
// dx[M,K] = dy[M,N] @ W[K,N]^T (+ epilogue)
static int linear_dgrad(const void* dy, int N, const void* W, int K, void* dx, int M, merlot_gemm_t extra, cudaStream_t st) {
  merlot_gemm_t g = extra;
  g.M = M; g.N = K; g.K = N;
  g.a = dy; g.lda = N; g.a_mn_major = 0;
  g.b = W; g.ldb = N; g.b_mn_major = 0;
  g.out = dx; g.ld_out = K;
  return merlot_gemm_bf16(&g, st);
}

#define RC(expr)            \
  do {                      \
    int _rc = (expr);       \
    if (_rc) return _rc;    \
  } while (0)

}  // namespace mb

using namespace mb;

extern "C" size_t merlot_stack_activation_bytes(const merlot_stack_t* s) {
  if (!s) return 0;
  const size_t M = (size_t)s->B * s->S;
  const size_t per = layer_act_bytes(s);
  return per * (s->save_for_backward ? (size_t)s->layers : 1) + align_up(M * 4) * 2;
}

extern "C" size_t merlot_stack_scratch_bytes(const merlot_stack_t* s) {
  if (!s) return 0;
  const size_t M = (size_t)s->B * s->S, H = s->H, I = s->I;
  return align_up(M * H * 2) * 4 + align_up(M * 3 * H * 2) + align_up(M * I * 2) +
         align_up(merlot_attention_bwd_workspace_bytes(s->B, s->S, s->heads)) +
         align_up((size_t)s->B * s->heads * s->S * 4) + align_up(merlot_layernorm_bwd_workspace_bytes(s->H));
}

extern "C" int merlot_stack_forward(const merlot_stack_t* s, void* stream_) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
  RC(check_stack(s));
  MB_REQUIRE(s->y != nullptr, MERLOT_EINVAL, "stack_forward: y is null");
  const int M = s->B * s->S, H = s->H, I = s->I;
  const size_t per = layer_act_bytes(s);
  char* arena = reinterpret_cast<char*>(s->act_arena);
  const size_t nlay_saved = s->save_for_backward ? (size_t)s->layers : 1;
  float* mean_f = reinterpret_cast<float*>(arena + per * nlay_saved);
  float* rstd_f = reinterpret_cast<float*>(arena + per * nlay_saved + align_up((size_t)M * 4));
  const void* h = s->h_in;
  for (int l = 0; l < s->layers; ++l) {
    const merlot_layer_params_t& P = s->layer_params[l];
    LayerAct A = carve(s, arena + (s->save_for_backward ? per * l : 0));
    // forward-only mode ping-pongs the residual stream between hmid/hout of the single saved layer: h (= previous hout)
    // is consumed by the out-proj epilogue before hout is rewritten by FFN2, so the aliasing is safe.
    RC(ln_fwd(h, A.x1, P.ln1_gamma, P.ln1_beta, A.mean1, A.rstd1, M, H, st));
    {
      merlot_gemm_t e = gemm_base(0, 0, 0);
      e.out = A.qkv; e.ld_out = 3 * H;
      RC(linear_fwd(A.x1, H, P.w_qkv, 3 * H, P.b_qkv, M, e, st));
    }
    {
      merlot_attn_t a;
      memset(&a, 0, sizeof(a));
      a.B = s->B; a.S = s->S; a.heads = s->heads; a.head_dim = 64; a.qkv = A.qkv; a.ld_qkv = 3 * H; a.valid = s->valid;
      a.pair_viz_len = s->pair_viz_len; a.pair_chunk_len = s->pair_chunk_len;
      a.scale = 0.125f; a.ctx = A.ctx; a.ld_ctx = H; a.lse = A.lse;
      // utils/transformer.py:114-115; the colsum / probs calls below see the same mask (self_attn_probs is post-dropout)
      a.dropout_p = s->attention_dropout_p; a.dropout_seed = s->dropout_seed; a.dropout_site = s->dropout_site_base + l;
      RC(merlot_attention_fwd(&a, st));
      if (s->attn_colsum) {
        a.colsum = s->attn_colsum;
        a.colsum2 = s->attn_colsum2; a.colsum_split = s->attn_colsum_split; a.colsum_valid_q = s->attn_colsum_valid_q;
        RC(merlot_attention_colsum(&a, st));
      }
      if (s->attn_probs) RC(merlot_attention_probs(&a, s->attn_probs + (size_t)l * s->B * s->S * s->S, st));
    }
    {
      merlot_gemm_t e = gemm_base(0, 0, 0);
      e.out = A.hmid; e.ld_out = H; e.resid = h; e.ld_resid = H;
      if (s->hidden_dropout_p > 0.f) {
        e.flags |= MERLOT_GEMM_DROPOUT; e.dropout_p = s->hidden_dropout_p; e.dropout_seed = s->dropout_seed;
        e.dropout_site = s->dropout_site_base + 2 * l;
      }
      RC(linear_fwd(A.ctx, H, P.w_o, H, P.b_o, M, e, st));
    }
    RC(ln_fwd(A.hmid, A.x2, P.ln2_gamma, P.ln2_beta, A.mean2, A.rstd2, M, H, st));
    {
      merlot_gemm_t e = gemm_base(0, 0, 0);
      e.out = A.pre; e.ld_out = I; e.out2 = A.act; e.ld_out2 = I; e.flags = MERLOT_GEMM_GELU;
      if (s->save_for_backward) e.flags |= MERLOT_GEMM_GELU_GRAD_OUT;  // `pre` then holds gelu'(pre): all the backward needs of it
      RC(linear_fwd(A.x2, H, P.w_1, I, P.b_1, M, e, st));
    }
    {
      merlot_gemm_t e = gemm_base(0, 0, 0);
      e.out = A.hout; e.ld_out = H; e.resid = A.hmid; e.ld_resid = H;
      if (s->hidden_dropout_p > 0.f) {
        e.flags |= MERLOT_GEMM_DROPOUT; e.dropout_p = s->hidden_dropout_p; e.dropout_seed = s->dropout_seed;
        e.dropout_site = s->dropout_site_base + 2 * l + 1;
      }
      RC(linear_fwd(A.act, I, P.w_2, H, P.b_2, M, e, st));
    }
    h = A.hout;
  }
  RC(ln_fwd(h, s->y, s->final_gamma, s->final_beta, mean_f, rstd_f, M, H, st));
  return MERLOT_OK;
}

extern "C" int merlot_stack_backward(const merlot_stack_t* s, void* stream_) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
  RC(check_stack(s));
  MB_REQUIRE(s->save_for_backward, MERLOT_EINVAL, "stack_backward: forward was not run with save_for_backward");
  MB_REQUIRE(s->dy && s->scratch && s->d_final_gamma && s->d_final_beta, MERLOT_EINVAL, "stack_backward: null pointer");
  const int M = s->B * s->S, H = s->H, I = s->I;
  const size_t per = layer_act_bytes(s);
  char* arena = reinterpret_cast<char*>(s->act_arena);
  float* mean_f = reinterpret_cast<float*>(arena + per * s->layers);
  float* rstd_f = reinterpret_cast<float*>(arena + per * s->layers + align_up((size_t)M * 4));
  // scratch carve-up
  char* p = reinterpret_cast<char*>(s->scratch);
  auto take = [&](size_t n) { char* r = p; p += align_up(n); return r; };
  char* dhA = take((size_t)M * H * 2);
  char* dhB = take((size_t)M * H * 2);
  char* dtmp = take((size_t)M * H * 2);   // dx of a sub-block / d_ctx
  char* dmask = take((size_t)M * H * 2);  // dropout-masked copy of the stream gradient
  char* dqkv = take((size_t)M * 3 * H * 2);
  char* dpre = take((size_t)M * I * 2);
  float* dq_acc = (float*)take(merlot_attention_bwd_workspace_bytes(s->B, s->S, s->heads));
  float* dsum = (float*)take((size_t)s->B * s->heads * s->S * 4);
  void* lnws = take(merlot_layernorm_bwd_workspace_bytes(H));
  if (merlot_attention_bwd_dq_parts(s->S) == 0)  // atomic mode: the single slice must start at zero (K3 hands it back zeroed)
    MB_CHECK_CUDA(cudaMemsetAsync(dq_acc, 0, (size_t)M * H * 4, st));

  WgradLane* lane = wgrad_lane(st);
  cudaStream_t wst = lane ? lane->stream : st;
  bool pending[4] = {false, false, false, false};  // wgrad i of the previous use still has to be waited for by its overwriter
  // wgrad i: ordered behind everything enqueued on the main stream so far; `done[i]` marks the end of its reads
  auto wgrad_on_lane = [&](int i, const void* x, int K, const void* dy, int N, float* dW) -> int {
    if (lane) {
      MB_CHECK_CUDA(cudaEventRecord(lane->ready[i], st));
      MB_CHECK_CUDA(cudaStreamWaitEvent(wst, lane->ready[i], 0));
    }
    int rc = linear_wgrad(x, K, dy, N, dW, M, wst);
    if (rc) return rc;
    if (lane) {
      MB_CHECK_CUDA(cudaEventRecord(lane->done[i], wst));
      pending[i] = true;
    }
    return MERLOT_OK;
  };
  auto wait_wgrad = [&](int i) -> int {  // the next main-stream kernel overwrites what wgrad i reads
    if (lane && pending[i]) {
      MB_CHECK_CUDA(cudaStreamWaitEvent(st, lane->done[i], 0));
      pending[i] = false;
    }
    return MERLOT_OK;
  };
  const bool drop = s->hidden_dropout_p > 0.f;
  // ln_bwd(dy, x, stats, gamma, dres) -> dx [+ dropout-masked copy + bias gradient of the linear layer that fed this
  // residual add]; `next_bias`/`next_site` describe that layer (nullptr: nobody consumes a masked copy)
  auto ln_bwd_f = [&](const void* dy_, const void* x_, const float* mean_, const float* rstd_, const float* gamma_, const void* dres_,
                      void* dx_, float* dgamma_, float* dbeta_, float* next_bias, uint32_t next_site) -> int {
    return merlot_layernorm_bwd_fused(dy_, x_, mean_, rstd_, gamma_, dres_, dx_, (drop && next_bias) ? dmask : nullptr, dgamma_,
                                      dbeta_, next_bias, lnws, M, H, (drop && next_bias) ? s->hidden_dropout_p : 0.f,
                                      s->dropout_seed, next_site, st);
  };
  char* dh = dhA;
  char* dh_other = dhB;
  // partial backward (bwd_lo/bwd_hi): the stream gradient is back in dhA after every complete layer (two swaps per layer), so
  // a call that resumes below the top layer simply continues from dhA
  const int l_hi = (s->bwd_hi > 0) ? s->bwd_hi : s->layers;
  const int l_lo = (s->bwd_hi > 0) ? s->bwd_lo : 0;
  MB_REQUIRE(0 <= l_lo && l_lo < l_hi && l_hi <= s->layers, MERLOT_EINVAL, "stack_backward: bad layer range [%d, %d)", l_lo, l_hi);
  if (l_hi == s->layers)
  {  // final LN; its output is the gradient of the last layer's FFN2 output
    LayerAct A = carve(s, arena + per * (s->layers - 1));
    const merlot_layer_params_t& PL = s->layer_params[s->layers - 1];
    RC(ln_bwd_f(s->dy, A.hout, mean_f, rstd_f, s->final_gamma, nullptr, dh, s->d_final_gamma, s->d_final_beta, PL.g_b_2,
                s->dropout_site_base + 2 * (s->layers - 1) + 1));
  }
  for (int l = l_hi - 1; l >= l_lo; --l) {
    const merlot_layer_params_t& P = s->layer_params[l];
    LayerAct A = carve(s, arena + per * l);
    const void* h_in = (l == 0) ? s->h_in : (const void*)carve(s, arena + per * (l - 1)).hout;
    // ---- FFN2: hout = hmid + drop(act W2 + b2);  d = dropout_bwd(dh) and db2 were produced by the LN backward above ----
    const void* d = drop ? (const void*)dmask : (const void*)dh;
    RC(wgrad_on_lane(0, A.act, I, d, H, P.g_w_2));
    RC(wait_wgrad(1));  // dpre is about to be rewritten: the previous layer's W1 wgrad has to be through with it
    {
      merlot_gemm_t e = gemm_base(0, 0, 0);
      e.flags = MERLOT_GEMM_MUL_AUX; e.aux = A.pre; e.ld_aux = I;  // A.pre = gelu'(pre), saved by the forward epilogue
      RC(linear_dgrad(d, H, P.w_2, I, dpre, M, e, st));
    }
    // ---- FFN1 ----
    RC(merlot_bias_grad(dpre, 0, I, M, I, P.g_b_1, 0.f, 0, 0, st));
    RC(wgrad_on_lane(1, A.x2, H, dpre, I, P.g_w_1));
    RC(linear_dgrad(dpre, I, P.w_1, H, dtmp, M, gemm_base(0, 0, 0), st));
    // ---- LN2: d_hmid = dh + LN'(dx2); also emits dropout_bwd(d_hmid) and db_o for the out-projection ----
    RC(wait_wgrad(0));  // it rewrites dmask / the other stream-gradient buffer
    RC(ln_bwd_f(dtmp, A.hmid, A.mean2, A.rstd2, P.ln2_gamma, dh, dh_other, P.g_ln2_gamma, P.g_ln2_beta, P.g_b_o,
                s->dropout_site_base + 2 * l));
    { char* t = dh; dh = dh_other; dh_other = t; }
    // ---- attention output projection: hmid = h + drop(ctx Wo + bo) ----
    d = drop ? (const void*)dmask : (const void*)dh;
    RC(wgrad_on_lane(2, A.ctx, H, d, H, P.g_w_o));
    RC(linear_dgrad(d, H, P.w_o, H, dtmp, M, gemm_base(0, 0, 0), st));  // d_ctx
    // ---- attention ----
    RC(wait_wgrad(3));  // dqkv is about to be rewritten: the previous layer's QKV wgrad has to be through with it
    {
      merlot_attn_t a;
      memset(&a, 0, sizeof(a));
      a.B = s->B; a.S = s->S; a.heads = s->heads; a.head_dim = 64; a.qkv = A.qkv; a.ld_qkv = 3 * H; a.valid = s->valid;
      a.pair_viz_len = s->pair_viz_len; a.pair_chunk_len = s->pair_chunk_len;
      a.scale = 0.125f; a.ctx = A.ctx; a.ld_ctx = H; a.lse = A.lse; a.d_ctx = dtmp; a.dsum = dsum; a.dq_accum = dq_acc;
      a.ld_dq = H; a.dqkv = dqkv; a.ld_dqkv = 3 * H; a.d_bias_qkv = P.g_b_qkv;  // bias gradient fused into the finish pass
      a.dropout_p = s->attention_dropout_p; a.dropout_seed = s->dropout_seed; a.dropout_site = s->dropout_site_base + l;
      RC(merlot_attention_bwd(&a, st));
    }
    // ---- QKV projection ----
    RC(wgrad_on_lane(3, A.x1, H, dqkv, 3 * H, P.g_w_qkv));
    RC(linear_dgrad(dqkv, 3 * H, P.w_qkv, H, dtmp, M, gemm_base(0, 0, 0), st));
    // ---- LN1: d_h_in = d_hmid + LN'(dx1); feeds the previous layer's FFN2 ----
    RC(wait_wgrad(2));  // it rewrites dmask / the other stream-gradient buffer
    void* dst = (l == 0 && s->dh_in) ? s->dh_in : (void*)dh_other;
    float* nb = (l > 0) ? s->layer_params[l - 1].g_b_2 : nullptr;
    RC(ln_bwd_f(dtmp, h_in, A.mean1, A.rstd1, P.ln1_gamma, dh, dst, P.g_ln1_gamma, P.g_ln1_beta, nb,
                l > 0 ? s->dropout_site_base + 2 * (l - 1) + 1 : 0));
    { char* t = dh; dh = dh_other; dh_other = t; }
  }
  for (int i = 0; i < 4; ++i) RC(wait_wgrad(i));  // join: every parameter gradient of these layers is final on the caller's stream
  return MERLOT_OK;
}
