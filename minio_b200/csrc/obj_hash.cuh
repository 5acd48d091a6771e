// obj_hash.cuh — the object hashes hash.Reader computes over a PutObject body besides the mergeable CRCs: MD5 for the ETag
// (internal/etag/reader.go:119-131), SHA-256 of a signed payload (x-amz-content-sha256, internal/hash/reader.go:177-180) and the
// SHA-1 / SHA-256 of x-amz-checksum-sha1 / -sha256 (internal/hash/checksum.go:282-291).  Each is a chain over 64-byte blocks that
// cannot be split, so the only parallelism is across messages: one thread per (message, algorithm) work item.  That pays only when
// a launch holds many messages, as a merged PUT batch of the coalescer does.
//
// A message is the concatenation of two segments of one device buffer (in a merged batch: a request's full erasure blocks and its
// short last block, which sit apart), each at any byte offset and of any length.  Full 64-byte blocks that lie inside one segment
// are read with 16-byte aligned loads and realigned with funnel shifts, the next block's loads issued before the current block is
// compressed; only the block that straddles the segment boundary and the final padding block(s) are assembled bytewise.  A load
// never touches a 16-byte granule that holds no message byte.
#pragma once
#include "whole_hash.cuh"

namespace mec {

constexpr int kSumAlgos = 3;       // 0 = MD5, 1 = SHA-1, 2 = SHA-256 (MEC_SUM_MD5 << a)
constexpr int kSumRecord = 96;     // MEC_SUM_BYTES: MD5 at +0, SHA-1 at +32, SHA-256 at +64
constexpr int kSumThreads = 32;    // one warp per CTA: the few warps of a launch spread over every SM
__host__ __device__ constexpr int sum_digest_len(int a) { return a == 0 ? 16 : a == 1 ? 20 : 32; }

// One (message, algorithm) item: segment 0 at base + off0, segment 1 at base + off1 (len1 may be 0); digest at out_base + out
struct SumWork {
  int64_t off0, len0, off1, len1;
  int64_t out;
  int32_t algo, pad;
};
struct SumParams {
  const uint8_t* base;
  const SumWork* work;  // sorted by (algo, length descending): a warp runs one algorithm over similar lengths
  int64_t nwork;
  uint8_t* out;
};

__device__ __forceinline__ uint32_t rotl32(uint32_t x, int n) { return __funnelshift_l(x, x, n); }

// ---- MD5 (RFC 1321): little-endian message words -------------------------------------------------------------------------------
__device__ __forceinline__ void md5_compress(uint32_t (&h)[4], const uint32_t (&w)[16]) {
  constexpr uint32_t K[64] = {
      0xd76aa478, 0xe8c7b756, 0x242070db, 0xc1bdceee, 0xf57c0faf, 0x4787c62a, 0xa8304613, 0xfd469501, 0x698098d8, 0x8b44f7af, 0xffff5bb1,
      0x895cd7be, 0x6b901122, 0xfd987193, 0xa679438e, 0x49b40821, 0xf61e2562, 0xc040b340, 0x265e5a51, 0xe9b6c7aa, 0xd62f105d, 0x02441453,
      0xd8a1e681, 0xe7d3fbc8, 0x21e1cde6, 0xc33707d6, 0xf4d50d87, 0x455a14ed, 0xa9e3e905, 0xfcefa3f8, 0x676f02d9, 0x8d2a4c8a, 0xfffa3942,
      0x8771f681, 0x6d9d6122, 0xfde5380c, 0xa4beea44, 0x4bdecfa9, 0xf6bb4b60, 0xbebfbc70, 0x289b7ec6, 0xeaa127fa, 0xd4ef3085, 0x04881d05,
      0xd9d4d039, 0xe6db99e5, 0x1fa27cf8, 0xc4ac5665, 0xf4292244, 0x432aff97, 0xab9423a7, 0xfc93a039, 0x655b59c3, 0x8f0ccc92, 0xffeff47d,
      0x85845dd1, 0x6fa87e4f, 0xfe2ce6e0, 0xa3014314, 0x4e0811a1, 0xf7537e82, 0xbd3af235, 0x2ad7d2bb, 0xeb86d391};
  constexpr int R[16] = {7, 12, 17, 22, 5, 9, 14, 20, 4, 11, 16, 23, 6, 10, 15, 21};
  uint32_t a = h[0], b = h[1], c = h[2], d = h[3];
#pragma unroll
  for (int i = 0; i < 64; i++) {
    uint32_t f;
    int g;
    if (i < 16) { f = d ^ (b & (c ^ d)); g = i; }
    else if (i < 32) { f = c ^ (d & (b ^ c)); g = (5 * i + 1) & 15; }
    else if (i < 48) { f = b ^ c ^ d; g = (3 * i + 5) & 15; }
    else { f = c ^ (b | ~d); g = (7 * i) & 15; }
    const uint32_t t = d;
    d = c; c = b;
    b = b + rotl32(a + f + K[i] + w[g], R[(i >> 4) * 4 + (i & 3)]);
    a = t;
  }
  h[0] += a; h[1] += b; h[2] += c; h[3] += d;
}

// ---- SHA-1 (FIPS 180-4): big-endian message words, expanded in place ------------------------------------------------------------
__device__ __forceinline__ void sha1_compress(uint32_t (&h)[5], uint32_t (&w)[16]) {
  uint32_t a = h[0], b = h[1], c = h[2], d = h[3], e = h[4];
#pragma unroll
  for (int i = 0; i < 80; i++) {
    if (i >= 16) w[i & 15] = rotl32(w[(i - 3) & 15] ^ w[(i - 8) & 15] ^ w[(i - 14) & 15] ^ w[i & 15], 1);
    uint32_t f, k;
    if (i < 20) { f = d ^ (b & (c ^ d)); k = 0x5a827999; }
    else if (i < 40) { f = b ^ c ^ d; k = 0x6ed9eba1; }
    else if (i < 60) { f = (b & c) | (d & (b | c)); k = 0x8f1bbcdc; }
    else { f = b ^ c ^ d; k = 0xca62c1d6; }
    const uint32_t t = rotl32(a, 5) + f + e + k + w[i & 15];
    e = d; d = c; c = rotl32(b, 30); b = a; a = t;
  }
  h[0] += a; h[1] += b; h[2] += c; h[3] += d; h[4] += e;
}

// The chaining state of algorithm A; block() takes the 16 message words as little-endian loads of the block's bytes
template <int A>
struct SumState {
  static constexpr int kWords = A == 0 ? 4 : A == 1 ? 5 : 8;
  uint32_t h[kWords];
  __device__ __forceinline__ void init() {
    if (A == 0) { h[0] = 0x67452301; h[1] = 0xefcdab89; h[2] = 0x98badcfe; h[3] = 0x10325476; }
    if (A == 1) { h[0] = 0x67452301; h[1] = 0xefcdab89; h[2] = 0x98badcfe; h[3] = 0x10325476; h[kWords - 1] = 0xc3d2e1f0; }
    if (A == 2) {
      const uint32_t iv[8] = {0x6a09e667, 0xbb67ae85, 0x3c6ef372, 0xa54ff53a, 0x510e527f, 0x9b05688c, 0x1f83d9ab, 0x5be0cd19};
#pragma unroll
      for (int i = 0; i < kWords; i++) h[i] = iv[i];
    }
  }
  __device__ __forceinline__ void block(uint32_t (&w)[16]) {
    if (A == 0) {
      md5_compress(reinterpret_cast<uint32_t(&)[4]>(h), w);
    } else {
#pragma unroll
      for (int i = 0; i < 16; i++) w[i] = bswap32(w[i]);
      if (A == 1) sha1_compress(reinterpret_cast<uint32_t(&)[5]>(h), w);
      else sha256_compress(reinterpret_cast<uint32_t(&)[8]>(h), w);
    }
  }
};

// 64 bytes starting `sh` (0..15) bytes into granule c[0] of the five 16-byte granules c[0..4], as 16 little-endian words
__device__ __forceinline__ void realign_block(uint32_t (&w)[16], const uint4 (&c)[5], uint32_t sh) {
  uint32_t u[20];
#pragma unroll
  for (int j = 0; j < 5; j++) { u[4 * j] = c[j].x; u[4 * j + 1] = c[j].y; u[4 * j + 2] = c[j].z; u[4 * j + 3] = c[j].w; }
  const uint32_t q = sh >> 2, r = 8 * (sh & 3);
  // whole-word shift by q in two selects (by 2, then by 1), then the byte shift r across word pairs
#pragma unroll
  for (int i = 0; i < 18; i++) u[i] = (q & 2) ? u[i + 2] : u[i];
#pragma unroll
  for (int i = 0; i < 17; i++) u[i] = (q & 1) ? u[i + 1] : u[i];
#pragma unroll
  for (int i = 0; i < 16; i++) w[i] = __funnelshift_r(u[i], u[i + 1], r);
}

// nb full 64-byte blocks contiguous from p (any alignment)
template <int A>
__device__ __forceinline__ void sum_run(SumState<A>& st, const uint8_t* p, int64_t nb) {
  if (nb <= 0) return;
  const uint4* g = reinterpret_cast<const uint4*>(reinterpret_cast<uintptr_t>(p) & ~static_cast<uintptr_t>(15));
  const uint32_t sh = static_cast<uint32_t>(reinterpret_cast<uintptr_t>(p) & 15);
  // block b covers granules 4b .. 4b+3, and 4b+4 when the start is misaligned (it is then block b+1's first granule)
  uint4 cur[5];
#pragma unroll
  for (int j = 0; j < 4; j++) cur[j] = __ldg(g + j);
  cur[4] = sh ? __ldg(g + 4) : make_uint4(0, 0, 0, 0);
  for (int64_t b = 0; b < nb; b++) {
    uint4 nxt[5] = {cur[4], cur[4], cur[4], cur[4], cur[4]};
    if (b + 1 < nb) {  // the next block's loads are in flight while this one is compressed
      const uint4* q = g + 4 * (b + 1);
      if (!sh) nxt[0] = __ldg(q);
#pragma unroll
      for (int j = 1; j < 4; j++) nxt[j] = __ldg(q + j);
      if (sh) nxt[4] = __ldg(q + 4);
    }
    uint32_t w[16];
    realign_block(w, cur, sh);
    st.block(w);
#pragma unroll
    for (int j = 0; j < 5; j++) cur[j] = nxt[j];
  }
}

// Message bytes [o, o + 64) of the two-segment message as little-endian words: bytes at or past `have` (counted from o) are the
// padding 0x80 (at exactly `have`) and zeros
__device__ __forceinline__ void sum_bytes(uint32_t (&w)[16], const uint8_t* s0, int64_t l0, const uint8_t* s1, int64_t o, int have) {
#pragma unroll
  for (int j = 0; j < 16; j++) {
    uint32_t v = 0;
#pragma unroll
    for (int t = 0; t < 4; t++) {
      const int pos = 4 * j + t;
      uint32_t x = 0;
      if (pos < have) x = o + pos < l0 ? s0[o + pos] : s1[o + pos - l0];
      else if (pos == have) x = 0x80;
      v |= x << (8 * t);
    }
    w[j] = v;
  }
}

// The whole two-segment message s0[0, l0) ++ s1[0, l1), padding and length included, into the freshly initialised `st`
template <int A>
__device__ __forceinline__ void sum_message(SumState<A>& st, const uint8_t* s0, int64_t l0, const uint8_t* s1, int64_t l1) {
  const int64_t total = l0 + l1;
  uint32_t w[16];
  sum_run(st, s0, l0 >> 6);
  int64_t o = l0 & ~static_cast<int64_t>(63);
  if ((l0 & 63) && total - o >= 64) {  // the block across the segment boundary
    sum_bytes(w, s0, l0, s1, o, 64);
    st.block(w);
    o += 64;
  }
  if (o >= l0) {
    const int64_t nb = (total - o) >> 6;
    sum_run(st, s1 + (o - l0), nb);
    o += nb * 64;
  }
  // the last 0..63 bytes, 0x80, zeros and the 64-bit bit length (little-endian for MD5, big-endian for the SHAs)
  const int rem = static_cast<int>(total - o);
  sum_bytes(w, s0, l0, s1, o, rem);
  if (rem >= 56) {
    st.block(w);
#pragma unroll
    for (int j = 0; j < 16; j++) w[j] = 0;
  }
  const uint64_t bits = static_cast<uint64_t>(total) * 8;
  if (A == 0) { w[14] = static_cast<uint32_t>(bits); w[15] = static_cast<uint32_t>(bits >> 32); }
  else { w[14] = bswap32(static_cast<uint32_t>(bits >> 32)); w[15] = bswap32(static_cast<uint32_t>(bits)); }
  st.block(w);
}

template <int A>
__device__ __forceinline__ void sum_item(const SumParams& p, const SumWork& wk) {
  SumState<A> st;
  st.init();
  sum_message(st, p.base + wk.off0, wk.len0, p.base + wk.off1, wk.len1);
  uint8_t* o8 = p.out + wk.out;  // any alignment: bytewise
#pragma unroll
  for (int i = 0; i < SumState<A>::kWords; i++)
#pragma unroll
    for (int t = 0; t < 4; t++) o8[4 * i + t] = static_cast<uint8_t>(st.h[i] >> (A == 0 ? 8 * t : 24 - 8 * t));
}

__global__ void __launch_bounds__(kSumThreads) stream_sums_kernel(const SumParams p) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * kSumThreads + threadIdx.x;
  if (i >= p.nwork) return;
  const SumWork wk = p.work[i];
  if (wk.algo == 0) sum_item<0>(p, wk);
  else if (wk.algo == 1) sum_item<1>(p, wk);
  else sum_item<2>(p, wk);
}

}  // namespace mec
