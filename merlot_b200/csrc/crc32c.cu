// K15 merlot_crc32c_multi: CRC-32C (Castagnoli) of many device byte ranges in one launch -- the per-tensor checksums of a
// TensorFlow V2 checkpoint, computed where the tensors already are instead of on one host thread.
//
// The CRC register update is linear over GF(2).  With raw(M) the register after feeding M into a zero register and
// x^(8k) the polynomial that advances a register through k zero bytes (multiplication mod P in the reflected representation),
//   crc32c(M) = raw(M) ^ (0xFFFFFFFF * x^(8|M|)) ^ 0xFFFFFFFF   and   raw(A || B) = raw(A) * x^(8|B|) ^ raw(B).
// So every piece of a segment contributes raw(piece) * x^(8 * bytes after the piece) to the segment's CRC, and the
// contributions are combined with XOR, which is commutative: pieces can be checksummed in any order by any thread and
// accumulated with atomicXor.  The result is exact integer arithmetic and does not depend on the launch shape.
//
// Work split: every segment is cut into chunks of kChunk bytes; one warp owns one chunk and each lane a contiguous kLane-byte
// sub-range of it, read with 16-byte loads after an unaligned head of at most 15 bytes and folded in with slicing-by-8 tables
// in shared memory.  The lanes' registers are advanced to the chunk's end by the precomputed x^(8 m kLane), XOR-reduced across
// the warp, and advanced to the segment's end by x^(8 D), the product of the x^(8 * 2^b) of D's set bits, one bit pair per
// lane.  The first chunk of a segment also adds the init / xor-out term.  The grid is persistent: each CTA walks the segment
// table in tiles, scans the tile's chunk counts and takes every (grid warps)-th chunk, so the host never needs the segment
// lengths that live in the device table.
#include "host_common.h"

namespace {

static_assert(sizeof(merlot_crc_seg_t) == 16, "merlot_crc_seg_t layout is part of the C ABI (_lib.py packs it from the header)");

constexpr uint32_t kPoly = 0x82F63B78u;  // reflected Castagnoli polynomial
constexpr uint32_t kOne = 0x80000000u;   // the polynomial 1 in the reflected representation
constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kLane = 1024;                   // bytes per lane (a multiple of 16: every lane of a chunk has the same alignment)
constexpr long long kChunk = 32LL * kLane;    // bytes per warp

// a * b mod P, both in the reflected representation (bit 31 = x^0)
__host__ __device__ constexpr uint32_t gf_mul(uint32_t a, uint32_t b) {
  uint32_t p = 0;
  for (int i = 0; i < 32; ++i) {
    if (a & (kOne >> i)) p ^= b;
    b = (b & 1u) ? (b >> 1) ^ kPoly : b >> 1;
  }
  return p;
}

struct Tables {
  uint32_t t[8][256];  // slicing-by-8: t[0] = the byte table, t[k][i] = t[k-1][i] advanced by one more zero byte
  uint32_t x8[64];     // x^(8 * 2^b) mod P
  uint32_t kl[32];     // x^(8 * m * kLane) mod P
};

constexpr Tables make_tables() {
  Tables T{};
  for (uint32_t i = 0; i < 256; ++i) {
    uint32_t c = i;
    for (int k = 0; k < 8; ++k) c = (c & 1u) ? (c >> 1) ^ kPoly : c >> 1;
    T.t[0][i] = c;
  }
  for (int k = 1; k < 8; ++k)
    for (int i = 0; i < 256; ++i) T.t[k][i] = (T.t[k - 1][i] >> 8) ^ T.t[0][T.t[k - 1][i] & 0xFFu];
  T.x8[0] = kOne >> 8;  // x^8
  for (int b = 1; b < 64; ++b) T.x8[b] = gf_mul(T.x8[b - 1], T.x8[b - 1]);
  for (int m = 0; m < 32; ++m) {
    uint32_t r = kOne;
    for (int b = 0; b < 20; ++b)
      if ((static_cast<unsigned long long>(m) * kLane >> b) & 1ull) r = gf_mul(r, T.x8[b]);
    T.kl[m] = r;
  }
  return T;
}

__device__ const Tables g_tables = make_tables();

struct Smem {
  Tables tab;
  const uint8_t* ptr[kThreads];
  long long len[kThreads];
  long long incl[kThreads];  // inclusive prefix of the tile's chunk counts
  long long wsum[kWarps];
};

__device__ __forceinline__ uint32_t step8(uint32_t c, uint32_t w0, uint32_t w1, const uint32_t (*t)[256]) {
  w0 ^= c;
  return t[7][w0 & 0xFFu] ^ t[6][(w0 >> 8) & 0xFFu] ^ t[5][(w0 >> 16) & 0xFFu] ^ t[4][w0 >> 24] ^
         t[3][w1 & 0xFFu] ^ t[2][(w1 >> 8) & 0xFFu] ^ t[1][(w1 >> 16) & 0xFFu] ^ t[0][w1 >> 24];
}

__device__ __forceinline__ uint32_t step1(uint32_t c, uint8_t b, const uint32_t (*t)[256]) {
  return t[0][(c ^ b) & 0xFFu] ^ (c >> 8);
}

// raw register of p[0 .. n) fed into a zero register
__device__ uint32_t crc_range(const uint8_t* p, int n, const uint32_t (*t)[256]) {
  uint32_t c = 0;
  int h = static_cast<int>((16u - (reinterpret_cast<uintptr_t>(p) & 15u)) & 15u);
  if (h > n) h = n;
  for (int i = 0; i < h; ++i) c = step1(c, __ldg(p + i), t);
  p += h;
  n -= h;
  const uint4* q = reinterpret_cast<const uint4*>(p);
  const int nv = n >> 4;
  int j = 0;
  for (; j + 4 <= nv; j += 4) {
    uint4 v[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) v[u] = __ldg(q + j + u);
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      c = step8(c, v[u].x, v[u].y, t);
      c = step8(c, v[u].z, v[u].w, t);
    }
  }
  for (; j < nv; ++j) {
    const uint4 v = __ldg(q + j);
    c = step8(c, v.x, v.y, t);
    c = step8(c, v.z, v.w, t);
  }
  for (int i = nv * 16; i < n; ++i) c = step1(c, __ldg(p + i), t);
  return c;
}

// x^(8 n) mod P on every lane of the warp: lane l contributes the factors of bits l and l + 32 of n
__device__ __forceinline__ uint32_t xpow8_warp(unsigned long long n, const uint32_t* x8, int lane) {
  uint32_t f = ((n >> lane) & 1ull) ? x8[lane] : kOne;
  if ((n >> (lane + 32)) & 1ull) f = gf_mul(f, x8[lane + 32]);
#pragma unroll
  for (int o = 16; o; o >>= 1) f = gf_mul(f, __shfl_xor_sync(0xFFFFFFFFu, f, o));
  return f;
}

// x^(8 n) mod P for n < 2^20 on one thread
__device__ __forceinline__ uint32_t xpow8_small(unsigned n, const uint32_t* x8) {
  uint32_t r = kOne;
  for (int b = 0; n; ++b, n >>= 1)
    if (n & 1u) r = gf_mul(r, x8[b]);
  return r;
}

// Chunk k of a segment: its contribution to the segment's CRC, XORed into *out by lane 0.
__device__ void chunk_crc(const uint8_t* seg, long long len, long long k, unsigned* out, const Tables& T, int lane) {
  const long long start = k * kChunk;
  const long long end = min(start + kChunk, len);
  const long long a = min(start + static_cast<long long>(lane) * kLane, end);
  const long long e = min(a + kLane, end);
  const uint32_t c = crc_range(seg + a, static_cast<int>(e - a), T.t);
  uint32_t t;
  if (end - start == kChunk)
    t = gf_mul(c, T.kl[31 - lane]);
  else  // the segment's last chunk: lanes may be short or empty
    t = c ? gf_mul(c, xpow8_small(static_cast<unsigned>(end - e), T.x8)) : 0u;
#pragma unroll
  for (int o = 16; o; o >>= 1) t ^= __shfl_xor_sync(0xFFFFFFFFu, t, o);
  uint32_t v = gf_mul(t, xpow8_warp(static_cast<unsigned long long>(len - end), T.x8, lane));
  if (k == 0) v ^= gf_mul(0xFFFFFFFFu, xpow8_warp(static_cast<unsigned long long>(len), T.x8, lane)) ^ 0xFFFFFFFFu;
  if (lane == 0 && v) atomicXor(out, v);
}

__global__ void __launch_bounds__(kThreads) crc32c_kernel(const merlot_crc_seg_t* __restrict__ segs, int n,
                                                          unsigned* __restrict__ out) {
  __shared__ Smem s;
  {
    const uint32_t* src = reinterpret_cast<const uint32_t*>(&g_tables);
    uint32_t* dst = reinterpret_cast<uint32_t*>(&s.tab);
    for (int i = threadIdx.x; i < static_cast<int>(sizeof(Tables) / 4); i += kThreads) dst[i] = src[i];
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long gw = static_cast<long long>(blockIdx.x) * kWarps + warp;
  const long long n_warps = static_cast<long long>(gridDim.x) * kWarps;
  long long base = 0;  // chunks of the segments before this tile
  for (int t0 = 0; t0 < n; t0 += kThreads) {
    const int i = t0 + threadIdx.x;
    long long len = 0;
    const uint8_t* ptr = nullptr;
    if (i < n) {
      len = segs[i].bytes;
      ptr = static_cast<const uint8_t*>(segs[i].ptr);
    }
    long long x = (len + kChunk - 1) / kChunk;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const long long y = __shfl_up_sync(0xFFFFFFFFu, x, o);
      if (lane >= o) x += y;
    }
    if (lane == 31) s.wsum[warp] = x;
    s.ptr[threadIdx.x] = ptr;
    s.len[threadIdx.x] = len;
    __syncthreads();
    for (int w = 0; w < warp; ++w) x += s.wsum[w];
    s.incl[threadIdx.x] = x;
    __syncthreads();
    const long long tot = s.incl[kThreads - 1];
    for (long long c = base + ((gw - base % n_warps) + n_warps) % n_warps; c < base + tot; c += n_warps) {
      const long long r = c - base;
      int lo = 0, hi = kThreads - 1;  // first segment of the tile whose inclusive prefix exceeds r
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (s.incl[mid] > r) hi = mid; else lo = mid + 1;
      }
      chunk_crc(s.ptr[lo], s.len[lo], r - (lo ? s.incl[lo - 1] : 0), out + t0 + lo, s.tab, lane);
    }
    base += tot;
    __syncthreads();
  }
}

}  // namespace

extern "C" int merlot_crc32c_multi(const merlot_crc_seg_t* segs_dev, int n, unsigned* crc_out_dev, void* stream_) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
  MB_REQUIRE(n >= 0, MERLOT_EINVAL, "crc32c_multi: n=%d", n);
  if (n == 0) return MERLOT_OK;
  MB_REQUIRE(segs_dev && crc_out_dev, MERLOT_EINVAL, "crc32c_multi: null pointer");
  static const int per_sm = [] {
    int b = 0;
    return cudaOccupancyMaxActiveBlocksPerMultiprocessor(&b, crc32c_kernel, kThreads, 0) == cudaSuccess && b > 0 ? b : 1;
  }();
  MB_CHECK_CUDA(cudaMemsetAsync(crc_out_dev, 0, sizeof(unsigned) * static_cast<size_t>(n), st));
  crc32c_kernel<<<static_cast<unsigned>(mb::device_sms() * per_sm), kThreads, 0, st>>>(segs_dev, n, crc_out_dev);
  MB_CHECK_LAUNCH();
  return MERLOT_OK;
}
