// K17: exact rank and top-k of rows of fp32 scores, the ranking half of frame <-> transcript retrieval
// (merlot_b200/retrieval_validate.py).  One CTA per row r, with p = s[r, pos[r]]:
//   greater[r] = #{j : s[r,j] > p},  ties[r] = #{j != pos[r] : s[r,j] == p},
//   topk_idx/topk_val[r, :k] = the k largest entries ordered by (score descending, index ascending).
// NaN is never greater, never equal and never in the top k; a NaN p sets greater = -1 (ties = 0), a pos outside [0, cols)
// sets greater = -2 (ties = 0).  Slots past the row's non-NaN entries get index -1 and value NaN.
//
// Every thread strides over the row with 128-bit loads (when ld and the base allow them; two in flight) and counts in
// integers.  Each warp keeps one sorted top-k list spread over its lanes (lane t holds entry t, t < k), so the warp's k-th
// entry is an exact threshold: a column is a candidate only if it ranks before it.  Candidates are inserted one at a time
// by the whole warp (a ballot finds the slot, a shuffle shifts the tail), so an insertion costs a few warp instructions and
// never diverges.  Warp 0 then merges the 8 warp lists in k rounds of a warp argmax.  Every comparison is under the total
// order (score descending, index ascending; indices are unique) and the counts are integer sums, so the output is exact and
// does not depend on which thread saw which column.
#include <math.h>

#include "host_common.h"

namespace mb {

constexpr int kRankThreads = 256;
constexpr int kRankWarps = kRankThreads / 32;
constexpr unsigned kFull = 0xffffffffu;

// (va, ia) ranks before (vb, ib): a larger score, or an equal one at a smaller index; index -1 marks an empty slot, which
// ranks after everything.
__device__ __forceinline__ bool rank_before(float va, int ia, float vb, int ib) {
  if (ia < 0) return false;
  if (ib < 0) return true;
  return va > vb || (va == vb && ia < ib);
}

// The warp's sorted list: lane t < k holds (v, i), entry t.  (tv, ti) is entry k - 1 on every lane.
struct WarpTopK {
  float v, tv;
  int i, ti;
};

// Every lane with `pass` offers its (x, j); the warp inserts the offers one by one (all lanes take part).
__device__ __forceinline__ void warp_offer(WarpTopK& w, bool pass, float x, int j, int k, int lane) {
  unsigned m = __ballot_sync(kFull, pass);
  while (m) {
    const int src = __ffs(m) - 1;
    m &= m - 1;
    const float cv = __shfl_sync(kFull, x, src);
    const int cj = __shfl_sync(kFull, j, src);
    const unsigned at = __ballot_sync(kFull, lane < k && rank_before(cv, cj, w.v, w.i));
    if (!at) continue;  // no longer ranks before the k-th entry
    const int slot = __ffs(at) - 1;
    const float uv = __shfl_up_sync(kFull, w.v, 1);
    const int ui = __shfl_up_sync(kFull, w.i, 1);
    if (lane > slot && lane < k) { w.v = uv; w.i = ui; }
    if (lane == slot) { w.v = cv; w.i = cj; }
    w.tv = __shfl_sync(kFull, w.v, k - 1);
    w.ti = __shfl_sync(kFull, w.i, k - 1);
  }
}

__device__ __forceinline__ void rank_visit(WarpTopK& w, bool in_row, float x, int j, float p, int& gt, int& eq, int k,
                                           int lane) {
  gt += in_row && x > p;
  eq += in_row && x == p;
  warp_offer(w, in_row && x == x && rank_before(x, j, w.tv, w.ti), x, j, k, lane);
}

__global__ void __launch_bounds__(kRankThreads) rank_topk_kernel(const float* __restrict__ scores, int cols, long long ld,
                                                                 const int* __restrict__ pos, int k, int vec4,
                                                                 int* __restrict__ greater, int* __restrict__ ties,
                                                                 int* __restrict__ topk_idx, float* __restrict__ topk_val) {
  __shared__ int s_cnt[2][kRankWarps];
  __shared__ float s_v[kRankWarps][32];
  __shared__ int s_i[kRankWarps][32];

  const int r = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float* row = scores + (size_t)r * ld;
  const int pr = pos[r];
  const bool pos_ok = pr >= 0 && pr < cols;
  const float p = pos_ok ? row[pr] : 0.f;

  int gt = 0, eq = 0;
  WarpTopK w{0.f, 0.f, -1, -1};
  // trip counts are block-uniform, so every lane of a warp reaches every ballot
  if (vec4) {
    const int n4 = cols >> 2;
    const float4* row4 = reinterpret_cast<const float4*>(row);
    for (int base = 0; base < n4; base += 2 * kRankThreads) {
      const int q0 = base + tid, q1 = q0 + kRankThreads;
      const bool in0 = q0 < n4, in1 = q1 < n4;
      const float4 a = in0 ? __ldg(row4 + q0) : make_float4(0.f, 0.f, 0.f, 0.f);
      const float4 b = in1 ? __ldg(row4 + q1) : make_float4(0.f, 0.f, 0.f, 0.f);
      rank_visit(w, in0, a.x, 4 * q0 + 0, p, gt, eq, k, lane);
      rank_visit(w, in0, a.y, 4 * q0 + 1, p, gt, eq, k, lane);
      rank_visit(w, in0, a.z, 4 * q0 + 2, p, gt, eq, k, lane);
      rank_visit(w, in0, a.w, 4 * q0 + 3, p, gt, eq, k, lane);
      rank_visit(w, in1, b.x, 4 * q1 + 0, p, gt, eq, k, lane);
      rank_visit(w, in1, b.y, 4 * q1 + 1, p, gt, eq, k, lane);
      rank_visit(w, in1, b.z, 4 * q1 + 2, p, gt, eq, k, lane);
      rank_visit(w, in1, b.w, 4 * q1 + 3, p, gt, eq, k, lane);
    }
    const int j = (n4 << 2) + tid;  // at most 3 columns past the last whole float4
    const bool in = j < cols;
    rank_visit(w, in, in ? __ldg(row + j) : 0.f, j, p, gt, eq, k, lane);
  } else {
    for (int base = 0; base < cols; base += 4 * kRankThreads) {
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int j = base + u * kRankThreads + tid;
        const bool in = j < cols;
        rank_visit(w, in, in ? __ldg(row + j) : 0.f, j, p, gt, eq, k, lane);
      }
    }
  }

  // integer counts: warp shuffles, then thread 0 over the warps
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    gt += __shfl_xor_sync(kFull, gt, o);
    eq += __shfl_xor_sync(kFull, eq, o);
  }
  if (lane == 0) { s_cnt[0][warp] = gt; s_cnt[1][warp] = eq; }
  s_v[warp][lane] = w.v;
  s_i[warp][lane] = lane < k ? w.i : -1;
  __syncthreads();
  if (tid == 0) {
    int g = 0, e = 0;
    for (int x = 0; x < kRankWarps; ++x) { g += s_cnt[0][x]; e += s_cnt[1][x]; }
    if (!pos_ok) { g = -2; e = 0; }
    else if (p != p) { g = -1; e = 0; }
    else e -= 1;  // s[r, pos] == p itself
    greater[r] = g;
    ties[r] = e;
  }
  if (warp != 0) return;
  // warp 0: k rounds of an argmax over the heads of the warp lists (lane l < kRankWarps reads list l); the winner advances
  int head = 0;
  for (int t = 0; t < k; ++t) {
    float bv = 0.f;
    int bi = -1, bl = lane;
    if (lane < kRankWarps && head < k) { bv = s_v[lane][head]; bi = s_i[lane][head]; }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(kFull, bv, o);
      const int oi = __shfl_xor_sync(kFull, bi, o);
      const int ol = __shfl_xor_sync(kFull, bl, o);
      if (rank_before(ov, oi, bv, bi) || (oi < 0 && bi < 0 && ol < bl)) { bv = ov; bi = oi; bl = ol; }
    }
    if (lane == 0) {
      topk_idx[(size_t)r * k + t] = bi;
      topk_val[(size_t)r * k + t] = bi < 0 ? __int_as_float(0x7fc00000) : bv;
    }
    if (lane == bl && bi >= 0) ++head;
  }
}

}  // namespace mb

using namespace mb;

extern "C" int merlot_rank_topk(const float* scores, int rows, int cols, long long ld, const int* pos, int k, int* greater,
                                int* ties, int* topk_idx, float* topk_val, void* stream_) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
  MB_REQUIRE(rows >= 0 && cols > 0 && ld >= cols && k >= 1 && k <= 32, MERLOT_ESHAPE,
             "rank_topk: need rows >= 0, cols > 0, ld >= cols and 1 <= k <= 32 (rows=%d, cols=%d, ld=%lld, k=%d)", rows, cols,
             ld, k);
  MB_REQUIRE(scores && pos && greater && ties && topk_idx && topk_val, MERLOT_EINVAL, "rank_topk: null pointer");
  if (rows == 0) return MERLOT_OK;
  const int vec4 = (ld % 4 == 0) && (reinterpret_cast<uintptr_t>(scores) % 16 == 0);
  rank_topk_kernel<<<rows, kRankThreads, 0, st>>>(scores, cols, ld, pos, k, vec4, greater, ties, topk_idx, topk_val);
  MB_CHECK_LAUNCH();
  return MERLOT_OK;
}
