// K14 merlot_frames_prepare: the per-pixel half of the reference's frame parser (model/dataloader.py:72-96), fused --
//   tf.image.convert_image_dtype(uint8 -> float32)                                   x = u8 * float32(1/255)
//   resize_and_pad(do_random_scale=True, resize_method='random') (utils/model_utils.py:855-940)
//     tf.image.resize_images(.., [sh, sw], method, align_corners=True) with TF 1.15's legacy kernels
//     (resize_bilinear / resize_nearest_neighbor / resize_bicubic / resize_area, half_pixel_centers=False), crop at (oy, ox),
//     pad_to_bounding_box(0, 0, Hd, Wd)
//   tf.where(is_finite(x), x, 0)                                                    (model/dataloader.py:83)
//   lightweight_image_augment(allowed_transforms='brightness,contrast') + clip to [0, 1] (utils/model_utils.py:758-835)
//   tf.cast(.., bfloat16)                                                           (model/dataloader.py:94-96), RNE
// All arithmetic is float32 in the source's operation order; every product and sum is an explicitly rounded intrinsic so
// that nvcc cannot contract it into an FMA the reference's CPU kernels do not execute.  Only the pixels inside the crop
// window are resized and nothing intermediate is written: each output pixel reads its source taps straight from the packed
// uint8 frames.
//
// The contrast transform needs the mean of the whole padded Hd x Wd image before any of its pixels can be written, so the
// work is two launches: a block-per-image reduction over the images that draw the contrast transform (the others return at
// once; recomputing their resize is cheaper than a grid-wide barrier or an fp32 image round trip through HBM), then one thread
// per output pixel of every image.
#include <cuda_bf16.h>
#include <math.h>

#include "host_common.h"

namespace {
using bf16 = __nv_bfloat16;

static_assert(sizeof(merlot_frame_t) == 56, "merlot_frame_t layout is part of the C ABI (_lib.py packs it from the header)");

constexpr int kStatsThreads = 512;
constexpr int kApplyThreads = 256;

__device__ __forceinline__ float fmul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float fadd(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float fsub(float a, float b) { return __fsub_rn(a, b); }

// CalculateResizeScale (image_resizer_state.h), align_corners=True
__device__ __forceinline__ float resize_scale(int in, int out) {
  return out > 1 ? __fdiv_rn((float)(in - 1), (float)(out - 1)) : __fdiv_rn((float)in, (float)out);
}

struct Src {
  const uint8_t* p;
  int h, w;
  // convert_image_dtype: a multiply by float32(1/255), not a divide
  __device__ __forceinline__ float at(int y, int x, int c) const {
    return fmul((float)p[((size_t)y * w + x) * 3 + c], 0.003921568859368563f);
  }
};

__device__ __forceinline__ int bound(int v, int n) { return min(n - 1, max(0, v)); }

// resize_bilinear_op.cc: compute_interpolation_weights (LegacyScaler) + compute_lerp
__device__ void bilinear(const Src& s, float hs, float ws, int ry, int rx, float v[3]) {
  const float iy = fmul((float)ry, hs), ix = fmul((float)rx, ws);
  const float fy = floorf(iy), fx = floorf(ix);
  const int y0 = max((int)fy, 0), y1 = min((int)ceilf(iy), s.h - 1);
  const int x0 = max((int)fx, 0), x1 = min((int)ceilf(ix), s.w - 1);
  const float ly = fsub(iy, fy), lx = fsub(ix, fx);
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float tl = s.at(y0, x0, c), tr = s.at(y0, x1, c), bl = s.at(y1, x0, c), br = s.at(y1, x1, c);
    const float top = fadd(tl, fmul(fsub(tr, tl), lx));
    const float bottom = fadd(bl, fmul(fsub(br, bl), lx));
    v[c] = fadd(top, fmul(fsub(bottom, top), ly));
  }
}

// resize_nearest_neighbor_op.cc, align_corners: min(roundf(y * scale), in - 1)
__device__ void nearest(const Src& s, float hs, float ws, int ry, int rx, float v[3]) {
  const int y = min((int)roundf(fmul((float)ry, hs)), s.h - 1);
  const int x = min((int)roundf(fmul((float)rx, ws)), s.w - 1);
#pragma unroll
  for (int c = 0; c < 3; ++c) v[c] = s.at(y, x, c);
}

// resize_bicubic_op.cc InitCoeffsTable(-0.75): entry 2*i + odd of the 1025-entry table, evaluated in double as the source
// does (x = i / 1024 as float, a = -0.75 as double) and rounded to float once.
__device__ __forceinline__ float cubic_coeff(int i, int odd) {
  const double a = -0.75;
  double x = (double)i / 1024.0;  // exact
  if (!odd)  // ((a + 2) * x - (a + 3)) * x * x + 1
    return __double2float_rn(__dadd_rn(__dmul_rn(__dmul_rn(__dsub_rn(__dmul_rn(a + 2.0, x), a + 3.0), x), x), 1.0));
  x = x + 1.0;  // exact; ((a * x - 5 * a) * x + 8 * a) * x - 4 * a
  return __double2float_rn(
      __dsub_rn(__dmul_rn(__dadd_rn(__dmul_rn(__dsub_rn(__dmul_rn(a, x), 5.0 * a), x), 8.0 * a), x), 4.0 * a));
}

// GetWeightsAndIndices<LegacyScaler, use_keys_cubic=false>
__device__ __forceinline__ void cubic_taps(float scale, int out_loc, int limit, float w[4], int idx[4]) {
  const float in_f = fmul((float)out_loc, scale);
  const float fl = floorf(in_f);
  const int in = (int)fl;
  const int off = __float2int_rn(fmul(fsub(in_f, fl), 1024.f));  // lrintf: round half to even
  w[0] = cubic_coeff(off, 1);
  w[1] = cubic_coeff(off, 0);
  w[2] = cubic_coeff(1024 - off, 0);
  w[3] = cubic_coeff(1024 - off, 1);
#pragma unroll
  for (int k = 0; k < 4; ++k) idx[k] = bound(in - 1 + k, limit);
}

// Interpolate1D: ((v0 w0 + v1 w1) + v2 w2) + v3 w3
__device__ __forceinline__ float interp4(const float w[4], float v0, float v1, float v2, float v3) {
  return fadd(fadd(fadd(fmul(v0, w[0]), fmul(v1, w[1])), fmul(v2, w[2])), fmul(v3, w[3]));
}

// interpolate_with_caching: along y at each of the four x taps, then along x
__device__ void bicubic(const Src& s, float hs, float ws, int ry, int rx, float v[3]) {
  float wy[4], wx[4];
  int iy[4], ix[4];
  cubic_taps(hs, ry, s.h, wy, iy);
  cubic_taps(ws, rx, s.w, wx, ix);
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    float col[4];
#pragma unroll
    for (int k = 0; k < 4; ++k)
      col[k] = interp4(wy, s.at(iy[0], ix[k], c), s.at(iy[1], ix[k], c), s.at(iy[2], ix[k], c), s.at(iy[3], ix[k], c));
    v[c] = interp4(wx, col[0], col[1], col[2], col[3]);
  }
}

// resize_area_op.cc: the contribution of cell i to the box [in0, in1)
__device__ __forceinline__ float area_weight(int i, float in0, float in1, float scale) {
  if ((float)i < in0) return (float)(i + 1) > in1 ? scale : fsub((float)(i + 1), in0);
  return (float)(i + 1) > in1 ? fsub(in1, (float)i) : 1.f;
}

// ResizeAreaOp::ComputeLoop + ComputePatchSumOf3Channels (indices clamped with BOUND)
__device__ void area(const Src& s, float hs, float ws, int ry, int rx, float v[3]) {
  const float norm = (float)(1.0 / (double)fmul(hs, ws));  // float scale = 1.0 / (height_scale * width_scale)
  const float y0f = fmul((float)ry, hs), y1f = fmul((float)(ry + 1), hs);
  const float x0f = fmul((float)rx, ws), x1f = fmul((float)(rx + 1), ws);
  const int ys = (int)floorf(y0f), ye = (int)ceilf(y1f);
  const int xs = (int)floorf(x0f), xe = (int)ceilf(x1f);
  const float xs_scale = area_weight(xs, x0f, x1f, ws), xe_scale = area_weight(xe - 1, x0f, x1f, ws);
  float sum[3] = {0.f, 0.f, 0.f};
  for (int i = ys; i < ye; ++i) {
    const int yy = bound(i, s.h);
    const float sy = area_weight(i, y0f, y1f, hs);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      float r = fmul(s.at(yy, bound(xs, s.w), c), xs_scale);
      if (xs + 1 != xe) {
        for (int x = xs + 1; x < xe - 1; ++x) r = fadd(r, s.at(yy, bound(x, s.w), c));
        r = fadd(r, fmul(s.at(yy, bound(xe - 1, s.w), c), xe_scale));
      }
      sum[c] = fadd(sum[c], fmul(r, sy));
    }
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) v[c] = fmul(sum[c], norm);
}

// Output pixel (y, x) of frame f after resize, crop, pad and where(isfinite); zero in the padding.
__device__ __forceinline__ void frame_pixel(const merlot_frame_t& f, const uint8_t* src, int y, int x, float v[3]) {
  const int ry = f.offset_y + y, rx = f.offset_x + x;
  v[0] = v[1] = v[2] = 0.f;
  if (ry >= f.scaled_h || rx >= f.scaled_w) return;  // pad_to_bounding_box(0, 0, Hd, Wd)
  const Src s{src + f.src_offset, f.src_h, f.src_w};
  const float hs = resize_scale(f.src_h, f.scaled_h), ws = resize_scale(f.src_w, f.scaled_w);
  switch (f.method) {  // TF1 ResizeMethod order
    case 0: bilinear(s, hs, ws, ry, rx, v); break;
    case 1: nearest(s, hs, ws, ry, rx, v); break;
    case 2: bicubic(s, hs, ws, ry, rx, v); break;
    default: area(s, hs, ws, ry, rx, v); break;
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) v[c] = isfinite(v[c]) ? v[c] : 0.f;
}

// Per-channel mean over the padded out_h x out_w image, for the frames that draw the contrast transform.
__global__ void __launch_bounds__(kStatsThreads) frames_mean_kernel(const merlot_frame_t* __restrict__ frames,
                                                                    const uint8_t* __restrict__ src, int out_h, int out_w,
                                                                    float* __restrict__ mean) {
  const merlot_frame_t f = frames[blockIdx.x];
  if (f.augment != MERLOT_FRAME_CONTRAST) return;
  float acc[3] = {0.f, 0.f, 0.f};
  const int npx = out_h * out_w;
  for (int p = threadIdx.x; p < npx; p += kStatsThreads) {
    float v[3];
    frame_pixel(f, src, p / out_w, p % out_w, v);
#pragma unroll
    for (int c = 0; c < 3; ++c) acc[c] += v[c];
  }
  __shared__ float red[kStatsThreads / 32][3];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    float a = acc[c];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
    if (lane == 0) red[warp][c] = a;
  }
  __syncthreads();
  if (threadIdx.x < 3) {
    float a = 0.f;
    for (int w = 0; w < kStatsThreads / 32; ++w) a += red[w][threadIdx.x];
    mean[blockIdx.x * 3 + threadIdx.x] = __fdiv_rn(a, (float)npx);  // reduce_mean = sum / count
  }
}

// One thread per output pixel: resize + crop + pad + where(isfinite) + augment + clip + bf16.
__global__ void __launch_bounds__(kApplyThreads) frames_apply_kernel(const merlot_frame_t* __restrict__ frames,
                                                                     const uint8_t* __restrict__ src, int out_h, int out_w,
                                                                     const float* __restrict__ mean, bf16* __restrict__ out) {
  const int p = blockIdx.x * kApplyThreads + threadIdx.x;
  if (p >= out_h * out_w) return;
  const int n = blockIdx.y;
  const merlot_frame_t f = frames[n];
  float v[3];
  frame_pixel(f, src, p / out_w, p % out_w, v);
  const float fac[3] = {f.factor_r, f.factor_g, f.factor_b};
  bf16* o = out + ((size_t)n * out_h * out_w + p) * 3;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    float x = v[c];
    if (f.augment == MERLOT_FRAME_BRIGHTNESS) {
      x = fmul(x, fac[c]);
    } else if (f.augment == MERLOT_FRAME_CONTRAST) {
      const float m = mean[n * 3 + c];
      x = fadd(fmul(fsub(x, m), fac[c]), m);
    }
    if (f.augment != MERLOT_FRAME_NO_AUGMENT) x = fminf(fmaxf(x, 0.f), 1.f);  // clip_by_value(., 0, 1)
    o[c] = __float2bfloat16_rn(x);
  }
}

}  // namespace

extern "C" int merlot_frames_prepare(const merlot_frame_t* frames_dev, int n, const void* src_u8, int out_h, int out_w,
                                     float* mean_ws, void* out_bf16, void* stream_) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
  MB_REQUIRE(frames_dev && src_u8 && mean_ws && out_bf16, MERLOT_EINVAL, "frames_prepare: null pointer");
  MB_REQUIRE(n > 0 && n <= 65535 && out_h > 0 && out_w > 0 && (long long)out_h * out_w < (1LL << 30), MERLOT_ESHAPE,
             "frames_prepare: bad shape n=%d out=%dx%d", n, out_h, out_w);
  frames_mean_kernel<<<(unsigned)n, kStatsThreads, 0, st>>>(frames_dev, (const uint8_t*)src_u8, out_h, out_w, mean_ws);
  MB_CHECK_LAUNCH();
  const dim3 grid((unsigned)mb::ceil_div(out_h * out_w, kApplyThreads), (unsigned)n);
  frames_apply_kernel<<<grid, kApplyThreads, 0, st>>>(frames_dev, (const uint8_t*)src_u8, out_h, out_w, mean_ws, (bf16*)out_bf16);
  MB_CHECK_LAUNCH();
  return MERLOT_OK;
}
