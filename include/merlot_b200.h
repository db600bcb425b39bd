/*
 * merlot_b200 -- C-ABI of the H100-native (sm_90a) implementation of MERLOT's dense forward/backward hot path.
 *
 * The reference (rowanz/merlot) has no FFI/operator layer: its boundary is the Python class `MerlotModel`
 * (model/modeling.py:47-668) plus `optimization.build_optimizer_from_config` (utils/optimization.py:11-30), both of
 * which only call stock TF ops.  This header is the operator layer a maintainer would bind instead of those TF ops;
 * every entry point cites the reference call site(s) whose arithmetic it replaces.  The Python mirror of the
 * reference surface lives in merlot_b200/modeling.py and binds this header with ctypes (see INTEGRATION.md).
 *
 * Conventions
 *  - plain pointers and sizes only; every pointer is a DEVICE pointer owned by the caller (PyTorch allocates);
 *    the library allocates nothing persistent.
 *  - `stream` is a cudaStream_t passed as void*; all work is stream-ordered and asynchronous.
 *  - return value: MERLOT_OK (0) or a negative MERLOT_E* code; merlot_last_error() gives a thread-local message.
 *  - matrices are row-major; `ld*` are leading dimensions in ELEMENTS; bf16 = 16-bit brain float, f32 = IEEE float.
 *  - "tokens" M = batch*seq rows of the flattened [M, H] residual stream, as in utils/transformer.py:185.
 */
#ifndef MERLOT_B200_H_
#define MERLOT_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MERLOT_OK 0
#define MERLOT_EINVAL (-1)   /* bad argument / null pointer / unsupported flag combination */
#define MERLOT_ESHAPE (-2)   /* shape or alignment constraint violated (mirrors the reference's ValueError/assert) */
#define MERLOT_ECUDA (-3)    /* CUDA runtime / driver error */
#define MERLOT_ENOTIMPL (-4) /* config key accepted by the reference but not yet provided here (raised loudly) */

/* Leave n SMs to concurrently running collectives (NCCL gradient all-reduce): the persistent kernels (K1, K3) size their grids to
 * (SM count - n) so that none of their CTAs has to queue behind a collective's CTA.  0 = use every SM (single-GPU default). */
void merlot_set_sm_reserve(int n);
const char* merlot_last_error(void);
int merlot_abi_version(void);
/* number of kernels this library has launched since the last reset (bench.py reports it as gpu_launches) */
long long merlot_launch_count(void);
void merlot_reset_launch_count(void);

/* ------------------------------------------------------------------------------------------------------------
 * K1: bf16 tensor-core GEMM (wgmma, TMA-fed, fp32 accumulation in registers) with fused epilogues.
 *     C[M,N] = epilogue( alpha * sum_k A(m,k) * B(n,k) )
 * Replaces every tf.layers.dense / tf.matmul on the hot path and their tf.gradients:
 *   utils/transformer.py:21-25 (q/k/v), :130-135 (context_projection_layer), :149-155 (intermediate + gelu),
 *   :157-161 (output); utils/vision_transformer.py:196-205 (patch-embed conv as im2col GEMM);
 *   model/modeling.py:28-42 (project_and_norm), :208-217 (lm_head + tied logits), :521 (contrastive logits),
 *   :582-595 (temporal head).
 * Operand storage:
 *   a_mn_major = 0 : A is stored [M][K] (lda >= K)     a_mn_major = 1 : A is stored [K][M] (lda >= M)
 *   b_mn_major = 0 : B is stored [N][K] (ldb >= K)     b_mn_major = 1 : B is stored [K][N] (ldb >= N)
 *   (a TF `kernel` [in,out] used in the forward pass is B with b_mn_major=1; the same buffer is the K-major B of the
 *    dgrad GEMM; wgrad uses both activations MN-major.)  lda/ldb must be multiples of 8 elements, bases 16B-aligned.
 * Epilogue, applied in this order per element (row m, column n):
 *   v = alpha*acc; v += bias[n]; if GELU: {pre=v; v=gelu_erf(v)}; if MUL_DGELU: v *= gelu_erf'(aux[m,n]);
 *   if DROPOUT: v = keep(m,n) ? v/(1-p) : 0; v += resid[m,n]; store.
 *   With GELU and out2 != NULL: out <- pre (bf16), out2 <- gelu(pre); with GELU_GRAD_OUT as well: out <- gelu_erf'(pre) instead
 *   of pre -- the factor the FFN2 dgrad needs, computed where exp(-pre^2/2) is already in a register -- and that dgrad then uses
 *   MUL_AUX (v *= aux[m,n], one multiply) instead of MUL_DGELU (v *= gelu_erf'(aux[m,n]), ~17 instructions per element in an
 *   epilogue that is issue-bound).
 *   ATOMIC: fp32 red.add into out (split-K wgrad accumulation; out must be pre-zeroed or hold the running sum).
 * ------------------------------------------------------------------------------------------------------------ */
#define MERLOT_GEMM_OUT_F32 1u
#define MERLOT_GEMM_ATOMIC 2u
#define MERLOT_GEMM_GELU 4u
#define MERLOT_GEMM_MUL_DGELU 8u
#define MERLOT_GEMM_DROPOUT 16u
#define MERLOT_GEMM_GELU_GRAD_OUT 32u
#define MERLOT_GEMM_MUL_AUX 64u

typedef struct merlot_gemm {
  int M, N, K;
  const void* a; int lda; int a_mn_major;
  const void* b; int ldb; int b_mn_major;
  void* out; int ld_out;          /* bf16 unless MERLOT_GEMM_OUT_F32 */
  void* out2; int ld_out2;        /* optional second bf16 output (post-GELU) */
  const float* bias;              /* [N] fp32 or NULL */
  const void* resid; int ld_resid;/* bf16 [M,N] or NULL */
  const void* aux; int ld_aux;    /* bf16 [M,N]: pre-activation for MUL_DGELU / the saved factor for MUL_AUX */
  float alpha;
  uint32_t flags;
  float dropout_p; uint64_t dropout_seed; uint32_t dropout_site;
  int splits;                     /* 0 = auto; >1 requires MERLOT_GEMM_ATOMIC */
  int block_n;                    /* 0 = auto; else 128, 192 or 256 (tuning / tests) */
} merlot_gemm_t;

int merlot_gemm_bf16(const merlot_gemm_t* g, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * K2/K3/K4: masked softmax attention, FlashAttention-tiled on wgmma (probabilities never materialised in HBM).
 * Replaces utils/transformer.py:98-127 (scores = q k^T / sqrt(d); scores*m - 1e10*(1-m); softmax; probs @ v), its
 * tf.gradients, and the column sums of `self_attn_probs` consumed by model/modeling.py:428 (mask_inputs).
 *  qkv   : bf16 [B*S, ld_qkv], columns [0,H)=q, [H,2H)=k, [2H,3H)=v with head h at column h*64 (the fused QKV GEMM out).
 *  valid : uint8 [B*S] token validity (input_id != 0, model/modeling.py:148,363) or NULL = all valid (ViT, :239 of
 *          utils/vision_transformer.py).  mask[q,k] = valid[q] & valid[k] (model/modeling.py:158).
 *  lse   : f32 [B, heads, S] log-sum-exp of the masked scaled scores (written by fwd, read by bwd / colsum).
 *  fwd   : ctx bf16 [B*S, ld_ctx] <- softmax(.) v
 *  bwd   : needs ctx, d_ctx (bf16 [B*S, ld_ctx]); writes dsum (scratch f32 [B,heads,S]) and dqkv bf16 [B*S, ld_dqkv].
 *          dq_accum is an fp32 workspace of merlot_attention_bwd_workspace_bytes(B,S,heads) bytes with row stride ld_dq (= H):
 *          for sequences of <= 4 key tiles (merlot_attention_bwd_dq_parts(S) > 0) every key tile stores its dQ partial into its
 *          own [B*S, ld_dq] slice (no atomics, bitwise reproducible, no initialisation needed); longer sequences red.add into
 *          ONE slice that MUST be zero on entry and is re-zeroed on exit;
 *          with d_bias_qkv != NULL the same pass adds colsum(dqkv) to it (bias gradient of the q/k/v tf.layers.dense).
 *  colsum: colsum[b,k] += (1/heads) * sum_q P[b,h,q,k]   (f32 [B,S]; caller zeroes it once per stack).
 *  With dropout_p > 0, P above is the dropped P o Z / (1 - p) wherever it multiplies v or is summed (see the fields below).
 * ------------------------------------------------------------------------------------------------------------ */
typedef struct merlot_attn {
  int B, S, heads, head_dim;
  const void* qkv; int ld_qkv;
  const void* valid;
  float scale;                 /* 1/sqrt(head_dim), utils/transformer.py:99-100 */
  void* ctx; int ld_ctx;
  float* lse;
  const void* d_ctx;
  float* dsum;
  float* dq_accum; int ld_dq;
  void* dqkv; int ld_dqkv;
  float* colsum;
  float* d_bias_qkv;           /* optional f32 [3H]: += column sums of dqkv (gradient of the fused q/k/v bias) */
  float* colsum2;              /* colsum only: queries >= colsum_split accumulate here instead of `colsum` (optional) */
  int colsum_split;
  int colsum_valid_q;          /* colsum only: 1 = padding queries contribute nothing (attention_log, modeling.py:192-193) */
  /* disable_pairwise_lang_attn (model/modeling.py:160-168): with pair_chunk_len > 0 (needs `valid`) position t < pair_viz_len
   * is a vision token (segment 0) and position t >= pair_viz_len belongs to language chunk (t - pair_viz_len) / pair_chunk_len;
   * query and key exchange attention iff they share a segment or either one is a vision token.  0 = every valid pair. */
  int pair_viz_len, pair_chunk_len;
  /* attention_probs_dropout_prob (utils/transformer.py:114-115): probs = dropout(softmax(.), p) before probs @ v, with the
   * counter-based mask keep(seed, site, b, h, q, k) of ptx.cuh `attn_dropout_words` (restated in tests/attn_dropout_oracle.py).
   * fwd, bwd, colsum and probs must get the same triple for one layer; lse stays that of the undropped softmax; colsum and
   * probs sum the DROPPED probabilities (self_attn_probs is built from them, transformer.py:138).  p must lie in [0, 1)
   * (else MERLOT_EINVAL before any launch); p = 0 runs exactly the dropout-free kernels. */
  float dropout_p; uint64_t dropout_seed; uint32_t dropout_site;
} merlot_attn_t;

int merlot_attention_fwd(const merlot_attn_t* a, void* stream);
int merlot_attention_bwd(const merlot_attn_t* a, void* stream);
int merlot_attention_bwd_dq_parts(int S);                          /* slices used by bwd for this S; 0 = atomic single slice */
size_t merlot_attention_bwd_workspace_bytes(int B, int S, int heads); /* bytes of dq_accum (ld_dq = heads*64) */
int merlot_attention_colsum(const merlot_attn_t* a, void* stream);
/* Export path (PREDICT): probs_bss f32 [B,S,S] <- head-mean probabilities of this layer = one layer of `self_attn_probs`
 * (utils/transformer.py:208-209,238 with compress_attn=True), recomputed from qkv + lse. */
int merlot_attention_probs(const merlot_attn_t* a, float* probs_bss, void* stream);
/* attention_log (model/modeling.py:186-203): out4 = {lang2lang, lang2viz, viz2lang, viz2viz} normalised block sums of the
 * layer/head/batch-mean attention map, from the two split column sums (queries in the viz piece / in the lang piece). */
int merlot_attention_log_blocks(const float* c_viz, const float* c_lang, const void* valid_u8, int B, int S, int P, float* out4,
                                void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * K5: LayerNorm (utils/model_utils.py:113-130): fp32 statistics over the last dim, biased variance, eps inside rsqrt,
 *     y = x*s - mean*s + beta with s = rsqrt(var+eps)*gamma.  One warp per row, 128-bit accesses.  H % 8 == 0, H <= 1024.
 *     Optional fused inverted dropout on y (utils/model_utils.py:335-349; used after `embed_norm`, modeling.py:293-294).
 *     Row remap (map_per > 0): logical row r is written to / read from row (r / map_per) * map_stride + map_off + r % map_per,
 *     which places the viz and lang pieces side by side in the joint sequence (the tf.concat at model/modeling.py:151).
 * ------------------------------------------------------------------------------------------------------------ */
typedef struct merlot_ln {
  const void* x; int x_f32; int ld_x;
  void* y; int y_f32; int ld_y;
  const float* gamma; const float* beta;
  float* mean; float* rstd;          /* optional saved statistics [rows] */
  long long rows; int H; float eps;
  int map_per, map_stride, map_off;  /* output row remap; map_per = 0 disables */
  float dropout_p; uint64_t dropout_seed; uint32_t dropout_site;
} merlot_ln_t;
int merlot_layernorm_fwd(const merlot_ln_t* d, void* stream);

/* dx = LN'(dy) (+ dres); dgamma += sum dy*xhat; dbeta += sum dy.  dy is read through the same row remap / dropout mask. */
typedef struct merlot_ln_bwd {
  const void* dy; int dy_f32; int ld_dy;
  const void* x; int x_f32; int ld_x;
  const float* mean; const float* rstd; const float* gamma;
  const void* dres; int ld_dres;     /* optional residual-stream gradient added to dx (same dtype as dx) */
  void* dx; int dx_f32; int ld_dx;
  float* dgamma; float* dbeta;       /* accumulated (+=) */
  void* workspace;                   /* merlot_layernorm_bwd_workspace_bytes(H) */
  long long rows; int H;
  int map_per, map_stride, map_off;
  float dropout_p; uint64_t dropout_seed; uint32_t dropout_site;
} merlot_ln_bwd_t;
size_t merlot_layernorm_bwd_workspace_bytes(int H);
int merlot_layernorm_bwd(const merlot_ln_bwd_t* d, void* stream);

/* Fused bf16 LayerNorm backward used inside the stacks (H % 8 == 0, H <= 1024, contiguous rows):
 *   dx = LN'(dy) + dres;  dmask = dropout_bwd(dx) (when dropout_p > 0);  dbias += colsum(dmask or dx) (when dbias != NULL);
 *   dgamma, dbeta accumulated.  dbias is the bias gradient of the tf.layers.dense whose output fed this residual add
 *   (utils/transformer.py:136,162), i.e. it replaces one merlot_dropout_apply + one merlot_bias_grad pass. */
int merlot_layernorm_bwd_fused(const void* dy, const void* x, const float* mean, const float* rstd, const float* gamma,
                               const void* dres, void* dx, void* dmask, float* dgamma, float* dbeta, float* dbias,
                               void* workspace, long long rows, int H, float dropout_p, uint64_t seed, uint32_t site,
                               void* stream);
/* bias gradient of a tf.layers.dense: out[n] += sum_m dy[m,n], optionally through the forward dropout mask */
int merlot_bias_grad(const void* dy, int dy_f32, int ld, long long rows, int N, float* out, float dropout_p,
                     uint64_t seed, uint32_t site, void* stream);
/* backward of utils/model_utils.py:335-349 dropout with the counter-based mask the forward epilogue used */
int merlot_dropout_apply(const void* x_bf16, int ld_x, void* y_bf16, int ld_y, long long rows, int N, float p, uint64_t seed,
                         uint32_t site, void* stream);
/* one_hot_gather (utils/model_utils.py:225-235) as a real gather, and its transpose (scatter-add) */
int merlot_gather_rows(const void* src, int src_f32, int ld_s, const int* idx, void* dst, int dst_f32, int ld_d, int n, int H,
                       void* stream);
int merlot_scatter_add_rows(const void* src, int src_f32, int ld_s, const int* idx, void* dst, int dst_f32, int ld_d, int n,
                            int H, float scale, void* stream);
/* erf-GeLU (utils/model_utils.py:96-110) and its derivative on small fp32 head tensors */
int merlot_gelu_f32(const float* x, float* y, long long n, void* stream);
int merlot_gelu_bwd_f32(const float* dy, const float* pre, float* dx, long long n, void* stream);
/* bfloat16_getter cast (utils/model_utils.py:572-602) */
int merlot_cast_f32_to_bf16(const float* x, void* y, long long n, void* stream);
int merlot_cast_bf16_to_f32(const void* x, float* y, long long n, void* stream);
/* tf.math.l2_normalize(axis=-1) (model/modeling.py:43).  inv f32 [rows] <- rsqrt(max(sum x^2, 1e-12)), negated on rows where the
 * clamp is active (sum x^2 < 1e-12); bwd reads |inv| and takes the clamped branch (dx = dy * |inv|) exactly on those rows. */
int merlot_l2norm_fwd(const float* x, float* y, float* inv, int rows, int H, void* stream);
int merlot_l2norm_bwd(const float* dy, const float* y, const float* inv, float* dx, int rows, int H, void* stream);
/* raw_cross_entropy_with_logits (utils/model_utils.py:313-332) + argmax accuracy; bwd: dlogits = coeff[r]*(softmax-onehot) */
int merlot_softmax_ce_fwd(const float* logits, int ld, const int* labels, int rows, int C, float* loss, float* lse,
                          float* correct, void* stream);
int merlot_softmax_ce_bwd(const float* logits, int ld, const int* labels, int rows, int C, const float* lse,
                          const float* coeff, void* dlogits, int dlogits_f32, int ld_d, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Transformer stack driver (utils/transformer.py:171-247 `transformer`, pre-LN; forward and explicit backward).
 * One call enqueues a whole 12-layer stack.  Used three times per pretraining step: ViT (vision_transformer.py:247),
 * language-only (modeling.py:370) and joint (modeling.py:173) -- the last two with the SAME layer_params (scope
 * `encoder`, AUTO_REUSE), whose gradients therefore accumulate.
 * Weights: bf16 copies in the reference's [in,out] layout (w_qkv is [H,3H] = query|key|value kernels side by side).
 * Gradients: fp32, accumulated (+=) into g_*; zero them once per step.
 * ------------------------------------------------------------------------------------------------------------ */
typedef struct merlot_layer_params {
  const float *ln1_gamma, *ln1_beta;      /* LayerNorm_attn_ln0 */
  const void* w_qkv; const float* b_qkv;  /* query_layer|key_layer|value_layer fused: [H,3H], [3H] */
  const void* w_o;   const float* b_o;    /* context_projection_layer [H,H] */
  const float *ln2_gamma, *ln2_beta;      /* LayerNorm_mlp_ln0 */
  const void* w_1;   const float* b_1;    /* intermediate [H,I] */
  const void* w_2;   const float* b_2;    /* output [I,H] */
  float *g_ln1_gamma, *g_ln1_beta, *g_w_qkv, *g_b_qkv, *g_w_o, *g_b_o, *g_ln2_gamma, *g_ln2_beta, *g_w_1, *g_b_1, *g_w_2, *g_b_2;
} merlot_layer_params_t;

typedef struct merlot_stack {
  int B, S, H, I, heads, layers;
  const merlot_layer_params_t* layer_params;   /* HOST array [layers] of device pointers */
  const float *final_gamma, *final_beta;       /* LayerNorm_ln_final */
  float *d_final_gamma, *d_final_beta;
  const void* valid;                           /* uint8 [B*S] or NULL */
  const void* h_in;                            /* bf16 [B*S, H] stack input */
  void* y;                                     /* bf16 [B*S, H] = LN_final(h_last) */
  void* act_arena;                             /* merlot_stack_activation_bytes() */
  int save_for_backward;                       /* 0: forward only (arena holds one layer) */
  /* hidden dropout of layer l draws sites base + 2l (out-projection) and base + 2l + 1 (FFN2); attention-probability dropout
   * draws site base + l in its own counter stream.  attention_dropout_p must lie in [0, 1) (else MERLOT_EINVAL). */
  float hidden_dropout_p; float attention_dropout_p; uint64_t dropout_seed; uint32_t dropout_site_base;
  float* attn_colsum;                          /* optional f32 [B,S]: += sum over layers,queries of head-mean probs */
  float* attn_colsum2; int attn_colsum_split; int attn_colsum_valid_q;  /* optional split by query piece (attention_log) */
  float* attn_probs;                           /* optional f32 [layers][B,S,S]: head-mean probabilities of every layer (export) */
  /* backward */
  const void* dy;                              /* bf16 [B*S, H] gradient wrt y */
  void* dh_in;                                 /* bf16 [B*S, H] gradient wrt h_in (optional) */
  void* scratch;                               /* merlot_stack_scratch_bytes() */
  /* partial backward: layers [bwd_lo, bwd_hi) are walked top-down in this call (0,0 = all).  A call with bwd_hi == layers
   * starts from dy (final LayerNorm); later calls continue from the gradient left in `scratch` by the previous one, so a
   * caller can start the gradient all-reduce of a layer group while the groups below it are still running. */
  int bwd_lo, bwd_hi;
  int pair_viz_len, pair_chunk_len;            /* disable_pairwise_lang_attn, see merlot_attn_t (0, 0 = off) */
} merlot_stack_t;

size_t merlot_stack_activation_bytes(const merlot_stack_t* s);
size_t merlot_stack_scratch_bytes(const merlot_stack_t* s);
int merlot_stack_forward(const merlot_stack_t* s, void* stream);
int merlot_stack_backward(const merlot_stack_t* s, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * K6/K7: token assembly around the stacks (see csrc/assemble.cu for the reference lines each one replaces).
 * ------------------------------------------------------------------------------------------------------------ */
int merlot_patch_im2col(const void* image_bf16_nhwc, void* a_bf16, int N, int H0, int W0, int P, void* stream);
int merlot_vit_assemble_fwd(const float* patch, const float* pos_table, const float* cls_emb, float* xsum, int N, int h1,
                            int w1, int ncls, int tab_w, int H, void* stream);
int merlot_vit_assemble_bwd(const float* dxsum, void* dpatch_bf16, int N, int np, int ncls, int H, void* stream);
int merlot_viz_assemble_fwd(const void* hv_bf16, const float* img_idx_pe, const int* img_idx, const float* final_pos,
                            const float* final_cls, float* xsum, float* img_trg, int N, int h1, int w1, int ncls, int sp,
                            int tab_w, int H, void* stream);
int merlot_viz_assemble_bwd(const float* dxsum, const float* d_img_trg, void* dhv_bf16, int N, int h1, int w1, int ncls,
                            int sp, int H, void* stream);
int merlot_embed_fwd(const int* ids, const float* emb, const float* pos, float* xsum, long long R, int L, int H, void* stream);
int merlot_group_rowsum(const float* src, int ld, int groups, int per, int t0, int nt, const int* idxmap, float* dst,
                        int ld_dst, int H, void* stream);
int merlot_segment_rowsum_scatter(const float* src, int ld, int n_seg, int per, const int* idx, float* dst, int ld_dst, int H,
                                  void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * K12: MerlotModel.mask_inputs (model/modeling.py:381-489) with the random draws injected by the caller
 * (gumbel = -log(-log(U)) of utils/model_utils.py:647; two SpanBERT categorical draws; the 10/80/10 option draw;
 * uniform replacement ids in [100, vocab)).  Bit-exact integer outputs.
 *  w_non = 0.01f, w_delta = float(topk_val - 0.01), logw_* = log of the two weights, w_max = reduce_max(mask_weight).
 * ------------------------------------------------------------------------------------------------------------ */
typedef struct merlot_mask {
  const int* ids; const float* attn_summ; const float* gumbel; const int* span_lower; const int* span_upper;
  const int* option; const int* rand_ids;
  int* masked_ids; int* masked_idx; void* valid_out;
  int B, L, num_topk, num_to_mask, do_spanbert, mask_token;
  float w_delta, w_non, logw_top, logw_non, w_max;
} merlot_mask_t;
int merlot_mask_inputs(const merlot_mask_t* m, void* stream);
/* The five random tensors of mask_inputs drawn on device (Philox keyed by seed): gumbel f32 [n_tok] = -log(-log U),
 * span_lower/upper int32 [n_span] ~ categorical(p_len0, p_len1, 1-p_len0-p_len1), option int32 [n_tok] ~ (0.1, 0.8, 0.1),
 * rand_ids int32 [n_tok] uniform in [100, vocab)  (model/modeling.py:445-481, utils/model_utils.py:640-649). */
int merlot_mask_draws(float* gumbel, int* span_lower, int* span_upper, int* option, int* rand_ids, long long n_tok, long long n_span,
                      int vocab, float p_len0, float p_len1, uint64_t seed, void* stream);
int merlot_ids_valid(const int* ids, void* valid_u8, long long n, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * K10: fused AdamW on a contiguous slice of the flat parameter arena (utils/optimization.py:339-416, :267-288).
 * lr_t = lr * schedule * sqrt(1-beta2^t)/(1-beta1^t) is computed by the host (optimization.py:352-358).
 * ------------------------------------------------------------------------------------------------------------ */
typedef struct merlot_adamw {
  float* p; float* g; void* m; void* v;   /* fp32 master, fp32 grad, bf16 m, packed bf16 v */
  void* p_bf16;                           /* optional bf16 compute copy of p */
  long long n;
  float beta1, one_minus_beta1, beta2, one_minus_beta2, epsilon, lr_t, weight_decay, grad_scale;
  int zero_grad;
} merlot_adamw_t;
int merlot_adamw_step(const merlot_adamw_t* d, void* stream);
/* tf.clip_by_global_norm over the flat gradient arena (utils/optimization.py:233-237); scratch_f64 = one device double;
 * norm_out (optional device float) receives the pre-clip global norm (the reference's gradnorms/_overall metric). */
int merlot_clip_by_global_norm(float* g, long long n, float clip_norm, double* scratch_f64, float* norm_out, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Loss-head glue (model/modeling.py:491-668): integer index/label construction and weighted reductions, on device.
 * ------------------------------------------------------------------------------------------------------------ */
/* is_valid of the joint sequence: viz part all true (modeling.py:106-107), lang part ids != 0 (:148) */
int merlot_joint_valid(const int* ids, void* valid_u8, int B, int P, int L, void* stream);
/* rows of the masked positions in the joint sequence and their targets (modeling.py:533-536) */
int merlot_mlm_index(const int* ids, const int* masked_idx, int* rows, int* targets, int B, int L, int k, int P, void* stream);
/* allpairs_temporal_labels (modeling.py:598-620) + the 0.01/1.0 pair weights (:635,649-650) */
int merlot_temporal_labels(const int* video_src_ids, const int* shuffled_idx_img, int* labels, float* weights, int B, int n,
                           void* stream);
/* out2[0] = sum(l*w)/denom, out2[1] = sum(correct*w)/(sum w + 1e-5); coeff[r] = scale*w[r]/denom.
 * denom_mode 0: denom = R (reduce_mean); 1: denom = sum w + 1e-5 (modeling.py:543).  w: weights, or labels != 0, or 1. */
int merlot_weighted_loss(const float* per_row_loss, const float* correct, const float* weights, const int* nz_labels, int R,
                         int denom_mode, float scale, float* out2, float* coeff, void* stream);
/* tiny strided fp32 matmul C = alpha * A B^T + beta * C for the contrastive logits (modeling.py:521) and their grads */
int merlot_small_gemm_f32(const float* A, long long sam, long long sak, const float* B, long long sbn, long long sbk, float* C,
                          int ldc, int M, int N, int K, float alpha, float beta, void* stream);
int merlot_axpby_f32(const float* x, float* y, long long n, float a, float b, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * K13: hybrid ResNet-lite stem, FORWARD pieces (utils/vision_transformer.py:8-170; what merlot.yaml's
 * `resnet_layers: [3, 4, 9]` selects).  Convolutions themselves are merlot_gemm_bf16 calls on the NHWC activation matrix
 * (1x1) or on the im2col matrix below (3x3); see csrc/stem.cu.
 * ------------------------------------------------------------------------------------------------------------ */
/* weight standardisation (:56-60): w fp32 [rows = kh*kw*cin, cout] -> bf16 [rows_pad, cout] (rows past `rows` zero) */
int merlot_ws_weights(const float* w, int rows, int rows_pad, int cout, void* out_bf16, void* stream);
/* 3x3 taps of an NHWC bf16 tensor with one ring of zero padding, stride 1 (SAME) or 2 (fixed_padding :8-19 + VALID);
 * out [N*ho*wo, ld], columns (ky, kx, c), columns >= 9*C zero; sub_half: subtract 0.5 from in-range pixels (:193) */
int merlot_im2col3x3(const void* x_bf16, int N, int h, int w, int C, int stride, int sub_half, void* out_bf16, int ld, void* stream);
/* batch_norm_relu (:22-27): GroupNorm(groups, eps) with one-pass moments (utils/model_utils.py:196-201), optional ReLU,
 * optional relu(y + shortcut) (:96).  stats: f32 scratch [N, groups, 2]. */
int merlot_group_norm_fwd(const void* x_bf16, const float* gamma, const float* beta, const void* shortcut_bf16, void* y_bf16,
                          float* stats, int N, int HW, int C, int groups, float eps, int relu, void* stream);
/* tf.nn.avg_pool2d(ksize 2, strides 2, 'SAME') on NHWC bf16 (:81,93,159) */
int merlot_avgpool2_same(const void* x_bf16, int N, int h, int w, int C, void* y_bf16, void* stream);

/* K13 backward pieces (tf.gradients of the same graph); tests/test_gpu_stem.py checks them op by op and through the whole
 * training step. */
/* GroupNorm(+ReLU, +shortcut) backward: g = dy * [y > 0]; dx, dshortcut (= g, optional), dgamma += , dbeta += ;
 * red: f32 scratch [N, groups, 2]; stats: what merlot_group_norm_fwd left for this site */
int merlot_group_norm_bwd(const void* dy_bf16, const void* x_bf16, const void* y_bf16, const float* stats, const float* gamma,
                          void* dx_bf16, void* dshortcut_bf16, float* dgamma, float* dbeta, float* red, int N, int HW, int C,
                          int groups, float eps, int relu, void* stream);
int merlot_avgpool2_same_bwd(const void* dy_bf16, int N, int h, int w, int C, void* dx_bf16, void* stream);
/* adjoint of merlot_im2col3x3: dx[N,h,w,C] = sum of the taps of dcol [N*ho*wo, ld] that read each pixel */
int merlot_col2im3x3(const void* dcol_bf16, int N, int h, int w, int C, int stride, int ld, void* dx_bf16, void* stream);
/* weight-standardisation backward: dw[rows, cout] += d(standardise)/dw applied to dws[rows(, ld), cout] */
int merlot_ws_weights_bwd(const float* dws, int ld_dws, const float* w, int rows, int cout, float* dw, void* stream);
/* The same two operators for EVERY conv kernel of the stem in one launch each (the standardised operands depend on the
 * parameters only; the gradients meet at the end of the stem's backward pass).  items_dev: device array; item i serves blocks
 * [block0_i, block0_{i+1}) with block0_0 = 0 and 32 output channels per block, n_blocks = sum ceil(cout_i / 32). */
typedef struct {
  const float* w;    /* fp32 [rows, cout] kernel (flattened HWIO) */
  void* out;         /* bf16 [rows_pad, cout] standardised operand (forward) */
  const float* dws;  /* fp32 [rows(, ld_dws), cout] gradient of the standardised operand (backward) */
  float* dw;         /* fp32 [rows, cout] accumulated kernel gradient (backward) */
  int rows, rows_pad, cout, ld_dws, block0, reserved;
} merlot_ws_item_t;
int merlot_ws_weights_multi(const merlot_ws_item_t* items_dev, int n_items, int n_blocks, void* stream);
int merlot_ws_weights_bwd_multi(const merlot_ws_item_t* items_dev, int n_items, int n_blocks, void* stream);
int merlot_add_bf16(const void* a, const void* b, void* out, long long n, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * K14: frame preparation of the pretraining input pipeline (model/dataloader.py:72-96): uint8 HWC RGB frames ->
 * convert_image_dtype -> resize_and_pad(do_random_scale=True, resize_method='random') (utils/model_utils.py:855-940; TF 1.15
 * legacy resize kernels, align_corners=True) -> where(isfinite) -> brightness or contrast augment + clip
 * (utils/model_utils.py:758-835) -> bf16 (RNE), all in float32 in the reference's operation order; see csrc/frames.cu.
 * The caller draws and plans every frame (sizes, offsets, method, transform, factors); one descriptor per frame, in a device
 * table.  src_u8: the frames packed back to back; out_bf16: [n, out_h, out_w, 3]; mean_ws: f32 scratch [n, 3].
 * Every descriptor must satisfy src_h, src_w, scaled_h, scaled_w >= 1, offset_y, offset_x >= 0, method in [0, 3],
 * augment in [0, 2] and src_offset + 3*src_h*src_w within src_u8 (the kernel reads them unchecked).
 * ------------------------------------------------------------------------------------------------------------ */
#define MERLOT_FRAME_NO_AUGMENT 0
#define MERLOT_FRAME_BRIGHTNESS 1 /* x * factor[c] */
#define MERLOT_FRAME_CONTRAST 2   /* (x - mean_c) * factor[c] + mean_c, mean over the padded image before augmenting */
typedef struct merlot_frame {
  long long src_offset;             /* byte offset of the frame's [src_h, src_w, 3] pixels in src_u8 */
  int src_h, src_w;                 /* decoded size */
  int scaled_h, scaled_w;           /* resize target (sh, sw) */
  int offset_y, offset_x;           /* crop origin in the resized image; rows/columns past it and past (sh, sw) are zero */
  int method;                       /* tf.image.ResizeMethod (TF1): 0 bilinear, 1 nearest, 2 bicubic, 3 area */
  int augment;                      /* MERLOT_FRAME_* */
  float factor_r, factor_g, factor_b;
  int reserved;
} merlot_frame_t;
int merlot_frames_prepare(const merlot_frame_t* frames_dev, int n, const void* src_u8, int out_h, int out_w, float* mean_ws,
                          void* out_bf16, void* stream);

/* bench.py roofline support: time every K1 launch with CUDA events on its own stream between begin/end.
 * end() synchronises the device and returns the summed duration (ms), algorithmic FLOPs (2*M*N*K) and launch count. */
void merlot_gemm_profile_begin(void);
int merlot_gemm_profile_end(double* total_ms, double* total_flops, long long* launches);

#ifdef __cplusplus
}
#endif
#endif /* MERLOT_B200_H_ */
