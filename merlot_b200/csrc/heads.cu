// Small kernels for the three loss heads (model/modeling.py:491-668): index/label construction (integer, bit-exact),
// weighted loss reductions with their backward coefficients, and a tiny strided fp32 matmul (the VCR head's logit moves;
// the contrastive head runs on K16, contrastive.cu).  None of these is performance critical (<0.1 % of a step); they exist so that the whole loss path
// stays on the device, stream-ordered, with no host round trip.
#include "host_common.h"
#include "ptx.cuh"

namespace mb {

// valid[b, 0:P] = 1 (img_mask all true, modeling.py:106-107); valid[b, P:P+L] = ids[b,l] != 0 (:148)
__global__ void joint_valid_kernel(const int* __restrict__ ids, uint8_t* __restrict__ valid, int B, int P, int L) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int Sj = P + L;
  if (i >= (long long)B * Sj) return;
  const int b = (int)(i / Sj), t = (int)(i % Sj);
  valid[i] = t < P ? 1 : (ids[(size_t)b * L + (t - P)] != 0);
}

// The same with an image mask (model/modeling.py:106-122,152): row b's vision part is ni images of `span` tokens each, and
// token t < ni*span is valid iff img_mask[b / nt, t / span] != 0 (the mask is tiled to the nt texts of an image group, then
// over each image's tokens); img_mask == null means every image is valid.  valid[b, ni*span + l] = ids[b, l] != 0.
__global__ void joint_valid_img_kernel(const int* __restrict__ ids, const uint8_t* __restrict__ img_mask, uint8_t* __restrict__ valid,
                                       int B, int nt, int ni, int span, int L) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int P = ni * span, Sj = P + L;
  if (i >= (long long)B * Sj) return;
  const int b = (int)(i / Sj), t = (int)(i % Sj);
  if (t < P)
    valid[i] = img_mask ? (img_mask[(size_t)(b / nt) * ni + t / span] != 0) : 1;
  else
    valid[i] = ids[(size_t)b * L + (t - P)] != 0;
}

// rows[b*k+m] = b*Sj + P + masked_idx[b,m]  (modeling.py:534 in joint-sequence coordinates); targets = input_ids there (:536)
__global__ void mlm_index_kernel(const int* __restrict__ ids, const int* __restrict__ masked_idx, int* __restrict__ rows,
                                 int* __restrict__ targets, int B, int L, int k, int P) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * k) return;
  const int b = i / k, l = masked_idx[i];
  rows[i] = b * (P + L) + P + l;
  targets[i] = ids[(size_t)b * L + l];
}

// allpairs_temporal_labels (modeling.py:598-620) and the easy-pair weights (:635,649-650); row = b*n*n + i*n + j
__global__ void temporal_labels_kernel(const int* __restrict__ video_src_ids, const int* __restrict__ shuffled_idx, int* __restrict__ labels,
                                       float* __restrict__ w, int B, int n) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= B * n * n) return;
  const int b = r / (n * n), i = (r / n) % n, j = r % n;
  const bool same = video_src_ids[b * n + i] == video_src_ids[b * n + j];
  const int lab = (i == j) ? 1 : (i < j ? 2 : 3);
  labels[r] = same ? lab : 0;
  const bool easy = (shuffled_idx[b * n + i] < 64) && (shuffled_idx[b * n + j] < 64);
  w[r] = __fadd_rn(__fmul_rn(easy ? 0.f : 1.f, 0.99f), 0.01f);
}

// Weighted loss reduction, single block.  weights: w[r] (or labels[r] != 0 when w == null and nz_labels != null, or 1).
//   denom_mode 0: loss = sum(l*w) / R           (tf.reduce_mean of the weighted loss, modeling.py:523,655)
//   denom_mode 1: loss = sum(l*w) / (sum w + 1e-5)   (modeling.py:543-545)
//   acc = sum(correct*w) / (sum w + 1e-5)      (modeling.py:549,659)
//   coeff[r] = scale * w[r] / denom            (d loss_total / d l_r)
//   out[0] = loss * out_scale ... out[1] = acc
__global__ void __launch_bounds__(256) weighted_loss_kernel(const float* __restrict__ l, const float* __restrict__ correct, const float* __restrict__ w,
                                                            const int* __restrict__ nz_labels, int R, int denom_mode, float scale,
                                                            float* __restrict__ out, float* __restrict__ coeff) {
  __shared__ float s0[256], s1[256], s2[256];
  float a = 0.f, c = 0.f, ws = 0.f;
  for (int r = threadIdx.x; r < R; r += 256) {
    const float wr = w ? w[r] : (nz_labels ? (nz_labels[r] != 0 ? 1.f : 0.f) : 1.f);
    a += l[r] * wr;
    if (correct) c += correct[r] * wr;
    ws += wr;
  }
  s0[threadIdx.x] = a; s1[threadIdx.x] = c; s2[threadIdx.x] = ws;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) { s0[threadIdx.x] += s0[threadIdx.x + o]; s1[threadIdx.x] += s1[threadIdx.x + o]; s2[threadIdx.x] += s2[threadIdx.x + o]; }
    __syncthreads();
  }
  const float denom = denom_mode == 0 ? (float)R : (s2[0] + 1e-5f);
  if (threadIdx.x == 0) {
    out[0] = s0[0] / denom;
    out[1] = s1[0] / (s2[0] + 1e-5f);
  }
  if (coeff)
    for (int r = threadIdx.x; r < R; r += 256) {
      const float wr = w ? w[r] : (nz_labels ? (nz_labels[r] != 0 ? 1.f : 0.f) : 1.f);
      coeff[r] = scale * wr / denom;
    }
}

// C[m,n] = alpha * sum_k A(m,k) * B(n,k) + beta * C[m,n], arbitrary element strides, one warp per output element
__global__ void small_gemm_kernel(const float* __restrict__ A, long long sam, long long sak, const float* __restrict__ Bm, long long sbn,
                                  long long sbk, float* __restrict__ Cm, int ldc, int M, int N, int K, float alpha, float beta) {
  const long long wid = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (wid >= (long long)M * N) return;
  const int m = (int)(wid / N), n = (int)(wid % N);
  float acc = 0.f;
  for (int k = lane; k < K; k += 32) acc += A[m * sam + k * sak] * Bm[n * sbn + k * sbk];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (lane == 0) {
    float* c = Cm + (size_t)m * ldc + n;
    *c = alpha * acc + (beta != 0.f ? beta * *c : 0.f);
  }
}

// y = a*x + b*y (fp32 vectors)
__global__ void axpby_kernel(const float* __restrict__ x, float* __restrict__ y, long long n, float a, float b) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) y[i] = a * x[i] + (b != 0.f ? b * y[i] : 0.f);
}

}  // namespace mb

using namespace mb;

extern "C" int merlot_joint_valid(const int* ids, void* valid, int B, int P, int L, void* stream_) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
  MB_REQUIRE(ids && valid, MERLOT_EINVAL, "joint_valid: null pointer");
  const long long n = (long long)B * (P + L);
  joint_valid_kernel<<<(unsigned)ceil_div_ll(n, 256), 256, 0, st>>>(ids, reinterpret_cast<uint8_t*>(valid), B, P, L);
  MB_CHECK_LAUNCH();
  return MERLOT_OK;
}

extern "C" int merlot_joint_valid_img(const int* ids, const void* img_mask, void* valid, int B, int nt, int ni, int span, int L,
                                      void* stream_) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
  MB_REQUIRE(ids && valid, MERLOT_EINVAL, "joint_valid_img: null pointer");
  MB_REQUIRE(B > 0 && nt > 0 && B % nt == 0 && ni > 0 && span > 0 && L >= 0, MERLOT_ESHAPE,
             "joint_valid_img: needs B > 0, nt > 0 dividing B, ni > 0, span > 0, L >= 0");
  const long long n = (long long)B * ((long long)ni * span + L);
  joint_valid_img_kernel<<<(unsigned)ceil_div_ll(n, 256), 256, 0, st>>>(ids, reinterpret_cast<const uint8_t*>(img_mask),
                                                                      reinterpret_cast<uint8_t*>(valid), B, nt, ni, span, L);
  MB_CHECK_LAUNCH();
  return MERLOT_OK;
}

extern "C" int merlot_mlm_index(const int* ids, const int* masked_idx, int* rows, int* targets, int B, int L, int k, int P,
                                void* stream_) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
  MB_REQUIRE(ids && masked_idx && rows && targets, MERLOT_EINVAL, "mlm_index: null pointer");
  mlm_index_kernel<<<ceil_div(B * k, 256), 256, 0, st>>>(ids, masked_idx, rows, targets, B, L, k, P);
  MB_CHECK_LAUNCH();
  return MERLOT_OK;
}

extern "C" int merlot_temporal_labels(const int* video_src_ids, const int* shuffled_idx_img, int* labels, float* weights, int B,
                                      int n, void* stream_) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
  MB_REQUIRE(video_src_ids && shuffled_idx_img && labels && weights, MERLOT_EINVAL, "temporal_labels: null pointer");
  temporal_labels_kernel<<<ceil_div(B * n * n, 256), 256, 0, st>>>(video_src_ids, shuffled_idx_img, labels, weights, B, n);
  MB_CHECK_LAUNCH();
  return MERLOT_OK;
}

extern "C" int merlot_weighted_loss(const float* per_row_loss, const float* correct, const float* weights, const int* nz_labels,
                                    int R, int denom_mode, float scale, float* out2, float* coeff, void* stream_) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
  MB_REQUIRE(per_row_loss && out2, MERLOT_EINVAL, "weighted_loss: null pointer");
  MB_REQUIRE(R > 0 && (denom_mode == 0 || denom_mode == 1), MERLOT_EINVAL, "weighted_loss: bad R/denom_mode");
  weighted_loss_kernel<<<1, 256, 0, st>>>(per_row_loss, correct, weights, nz_labels, R, denom_mode, scale, out2, coeff);
  MB_CHECK_LAUNCH();
  return MERLOT_OK;
}

extern "C" int merlot_small_gemm_f32(const float* A, long long sam, long long sak, const float* B, long long sbn, long long sbk,
                                     float* C, int ldc, int M, int N, int K, float alpha, float beta, void* stream_) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
  MB_REQUIRE(A && B && C, MERLOT_EINVAL, "small_gemm_f32: null pointer");
  MB_REQUIRE(M > 0 && N > 0 && K > 0 && (long long)M * N <= (1 << 22), MERLOT_ESHAPE, "small_gemm_f32: meant for tiny outputs (M*N <= 4M)");
  const long long threads = (long long)M * N * 32;
  small_gemm_kernel<<<(unsigned)ceil_div_ll(threads, 256), 256, 0, st>>>(A, sam, sak, B, sbn, sbk, C, ldc, M, N, K, alpha, beta);
  MB_CHECK_LAUNCH();
  return MERLOT_OK;
}

extern "C" int merlot_axpby_f32(const float* x, float* y, long long n, float a, float b, void* stream_) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
  MB_REQUIRE(x && y, MERLOT_EINVAL, "axpby_f32: null pointer");
  if (n == 0) return MERLOT_OK;
  axpby_kernel<<<(unsigned)ceil_div_ll(n, 256), 256, 0, st>>>(x, y, n, a, b);
  MB_CHECK_LAUNCH();
  return MERLOT_OK;
}
