// whole_hash.cuh — legacy whole-file bitrot algorithms (cmd/bitrot-whole.go:35-45, cmd/bitrot.go:47-64):
// SHA-256, BLAKE2b-512 and non-streaming HighwayHash-256 over a whole shard file.  These hashes chain over
// every erasure block of one shard file, so the only parallelism is across shard files (n per object,
// times the objects in a batch): one thread per stream, 16-byte aligned loads from a gathered, contiguous
// copy of each shard file.  MinIO's default since 2019 is the streaming HighwayHash256S handled by the
// fused kernel; this path exists for format compatibility (and BASELINE config 5), not for speed.
#pragma once
#include "ec_device.cuh"

namespace mec {

// ---- gather: shard file i of an object = concat over blocks b of shard (b, i) --------------------------
struct GatherParams {
  const uint8_t* src;      // object bytes (Split layout), block b at b*block_size
  const uint8_t* parity;   // parity shard (b, j) at parity + (b*m + j)*parity_pitch
  int64_t parity_pitch, block_size, len;
  int k, m;
  int64_t S;               // full shard size
  uint8_t* files;          // shard file i at files + i*file_pitch
  int64_t file_pitch, file_len;
};

__global__ void gather_shard_files_kernel(const GatherParams p) {
  const int i = blockIdx.y;  // shard index
  const int64_t nfull = p.len / p.block_size, tail = p.len % p.block_size;
  const int64_t St = (tail + p.k - 1) / p.k;
  for (int64_t o = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; o < p.file_len;
       o += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    int64_t b = o / p.S, x = o - b * p.S;
    int64_t per = p.S, blen = p.block_size;
    if (b >= nfull) { b = nfull; x = o - nfull * p.S; per = St; blen = tail; }
    uint8_t v = 0;
    if (i < p.k) {
      const int64_t off = static_cast<int64_t>(i) * per + x;
      if (off < blen) v = p.src[b * p.block_size + off];
    } else {
      v = p.parity[(b * p.m + (i - p.k)) * p.parity_pitch + x];
    }
    p.files[i * p.file_pitch + o] = v;
  }
}

// ---- SHA-256 ---------------------------------------------------------------------------------------------
__device__ __constant__ uint32_t kSha256K[64] = {
    0x428a2f98, 0x71374491, 0xb5c0fbcf, 0xe9b5dba5, 0x3956c25b, 0x59f111f1, 0x923f82a4, 0xab1c5ed5, 0xd807aa98, 0x12835b01, 0x243185be,
    0x550c7dc3, 0x72be5d74, 0x80deb1fe, 0x9bdc06a7, 0xc19bf174, 0xe49b69c1, 0xefbe4786, 0x0fc19dc6, 0x240ca1cc, 0x2de92c6f, 0x4a7484aa,
    0x5cb0a9dc, 0x76f988da, 0x983e5152, 0xa831c66d, 0xb00327c8, 0xbf597fc7, 0xc6e00bf3, 0xd5a79147, 0x06ca6351, 0x14292967, 0x27b70a85,
    0x2e1b2138, 0x4d2c6dfc, 0x53380d13, 0x650a7354, 0x766a0abb, 0x81c2c92e, 0x92722c85, 0xa2bfe8a1, 0xa81a664b, 0xc24b8b70, 0xc76c51a3,
    0xd192e819, 0xd6990624, 0xf40e3585, 0x106aa070, 0x19a4c116, 0x1e376c08, 0x2748774c, 0x34b0bcb5, 0x391c0cb3, 0x4ed8aa4a, 0x5b9cca4f,
    0x682e6ff3, 0x748f82ee, 0x78a5636f, 0x84c87814, 0x8cc70208, 0x90befffa, 0xa4506ceb, 0xbef9a3f7, 0xc67178f2};

__device__ __forceinline__ uint32_t rotr32(uint32_t x, int n) { return __funnelshift_r(x, x, n); }
__device__ __forceinline__ uint32_t bswap32(uint32_t x) { return prmt(x, 0u, 0x0123u); }

__device__ __forceinline__ void sha256_compress(uint32_t (&h)[8], uint32_t (&w)[16]) {  // w: big-endian message words
  uint32_t a = h[0], b = h[1], c = h[2], d = h[3], e = h[4], f = h[5], g = h[6], hh = h[7];
#pragma unroll
  for (int i = 0; i < 64; i++) {
    if (i >= 16) {
      const uint32_t w15 = w[(i - 15) & 15], w2 = w[(i - 2) & 15];
      const uint32_t s0 = rotr32(w15, 7) ^ rotr32(w15, 18) ^ (w15 >> 3);
      const uint32_t s1 = rotr32(w2, 17) ^ rotr32(w2, 19) ^ (w2 >> 10);
      w[i & 15] = w[i & 15] + s0 + w[(i - 7) & 15] + s1;
    }
    const uint32_t S1 = rotr32(e, 6) ^ rotr32(e, 11) ^ rotr32(e, 25);
    const uint32_t ch = (e & f) ^ (~e & g);
    const uint32_t t1 = hh + S1 + ch + kSha256K[i] + w[i & 15];
    const uint32_t S0 = rotr32(a, 2) ^ rotr32(a, 13) ^ rotr32(a, 22);
    const uint32_t mj = (a & b) ^ (a & c) ^ (b & c);
    hh = g; g = f; f = e; e = d + t1; d = c; c = b; b = a; a = t1 + S0 + mj;
  }
  h[0] += a; h[1] += b; h[2] += c; h[3] += d; h[4] += e; h[5] += f; h[6] += g; h[7] += hh;
}

// ---- BLAKE2b-512 (unkeyed) ------------------------------------------------------------------------------
__device__ __constant__ uint64_t kB2IV[8] = {0x6a09e667f3bcc908ull, 0xbb67ae8584caa73bull, 0x3c6ef372fe94f82bull, 0xa54ff53a5f1d36f1ull,
                                             0x510e527fade682d1ull, 0x9b05688c2b3e6c1full, 0x1f83d9abfb41bd6bull, 0x5be0cd19137e2179ull};
__device__ __constant__ uint8_t kB2Sigma[12][16] = {
    {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15}, {14, 10, 4, 8, 9, 15, 13, 6, 1, 12, 0, 2, 11, 7, 5, 3},
    {11, 8, 12, 0, 5, 2, 15, 13, 10, 14, 3, 6, 7, 1, 9, 4}, {7, 9, 3, 1, 13, 12, 11, 14, 2, 6, 5, 10, 4, 0, 15, 8},
    {9, 0, 5, 7, 2, 4, 10, 15, 14, 1, 11, 12, 6, 8, 3, 13}, {2, 12, 6, 10, 0, 11, 8, 3, 4, 13, 7, 5, 15, 14, 1, 9},
    {12, 5, 1, 15, 14, 13, 4, 10, 0, 7, 6, 3, 9, 2, 8, 11}, {13, 11, 7, 14, 12, 1, 3, 9, 5, 0, 15, 4, 8, 6, 2, 10},
    {6, 15, 14, 9, 11, 3, 0, 8, 12, 2, 13, 7, 1, 4, 10, 5}, {10, 2, 8, 4, 7, 6, 1, 5, 15, 11, 9, 14, 3, 12, 13, 0},
    {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15}, {14, 10, 4, 8, 9, 15, 13, 6, 1, 12, 0, 2, 11, 7, 5, 3}};
__device__ __forceinline__ uint64_t rotr64(uint64_t x, int n) { return (x >> n) | (x << (64 - n)); }
__device__ inline void blake2b_compress(uint64_t (&h)[8], const uint64_t (&m)[16], uint64_t t0, bool last) {
  uint64_t v[16];
#pragma unroll
  for (int i = 0; i < 8; i++) { v[i] = h[i]; v[i + 8] = kB2IV[i]; }
  v[12] ^= t0;
  if (last) v[14] = ~v[14];
#define MEC_B2G(a, b, c, d, x, y)                                                                       \
  do { a = a + b + x; d = rotr64(d ^ a, 32); c = c + d; b = rotr64(b ^ c, 24);                          \
       a = a + b + y; d = rotr64(d ^ a, 16); c = c + d; b = rotr64(b ^ c, 63); } while (0)
#pragma unroll 1
  for (int r = 0; r < 12; r++) {
    const uint8_t* s = kB2Sigma[r];
    MEC_B2G(v[0], v[4], v[8], v[12], m[s[0]], m[s[1]]);
    MEC_B2G(v[1], v[5], v[9], v[13], m[s[2]], m[s[3]]);
    MEC_B2G(v[2], v[6], v[10], v[14], m[s[4]], m[s[5]]);
    MEC_B2G(v[3], v[7], v[11], v[15], m[s[6]], m[s[7]]);
    MEC_B2G(v[0], v[5], v[10], v[15], m[s[8]], m[s[9]]);
    MEC_B2G(v[1], v[6], v[11], v[12], m[s[10]], m[s[11]]);
    MEC_B2G(v[2], v[7], v[8], v[13], m[s[12]], m[s[13]]);
    MEC_B2G(v[3], v[4], v[9], v[14], m[s[14]], m[s[15]]);
  }
#undef MEC_B2G
#pragma unroll
  for (int i = 0; i < 8; i++) h[i] ^= v[i] ^ v[i + 8];
}

// ---- one thread per stream; streams are contiguous, 16-byte aligned, padded with >= 128 readable bytes ------
// One stream of a launch with a stream table: data + off, len bytes (a merged batch of shard files of different lengths)
struct WholeStream {
  int64_t off, len;
};

// A launch hashes up to kWholeGroups algorithm groups: group g is streams [gstream[g], gstream[g+1]) of algorithm galgo[g], run by
// the threads from gthread[g] on (a multiple of 32: no warp runs two algorithms, and HighwayHash lane pairs stay in one warp).  A
// merged verification (mec_bitrot_verify_parts, mec_batcher_verify) mixes parts of every era in one launch, which then lasts as long
// as its longest file rather than the sum of one launch per algorithm.
constexpr int kWholeGroups = 3;

struct WholeHashParams {
  const uint8_t* data;   // stream s at data + s*pitch
  int64_t pitch, len;    // every stream has the same length
  const WholeStream* streams;  // device, optional: stream s is data + streams[s].off, streams[s].len bytes (pitch, len unused)
  int ngroups;
  int galgo[kWholeGroups];        // MEC_SHA256 = 1, MEC_HIGHWAYHASH256 = 2, MEC_BLAKE2B512 = 4
  int gstream[kWholeGroups + 1];  // group g = streams [gstream[g], gstream[g + 1])
  int gthread[kWholeGroups];      // first thread of group g
  uint8_t* out;          // digest of stream s at out + s*64
  uint64_t key[4];
};

__device__ __forceinline__ WholeStream whole_stream(const WholeHashParams& p, int s) {
  return p.streams ? p.streams[s] : WholeStream{static_cast<int64_t>(s) * p.pitch, p.len};
}

__global__ void whole_hash_kernel(const WholeHashParams p) {
  const int tid = blockIdx.x * blockDim.x + threadIdx.x;
  // the group of this thread's warp, from the warp's first thread
  // (static indices only: a run-time index into the parameters would copy them to the stack)
  const int warp0 = tid & ~31;
  int algo = p.galgo[0], first = p.gstream[0], end = p.gstream[1], local = tid - p.gthread[0];
#pragma unroll
  for (int q = 1; q < kWholeGroups; q++)
    if (q < p.ngroups && warp0 >= p.gthread[q]) { algo = p.galgo[q]; first = p.gstream[q]; end = p.gstream[q + 1]; local = tid - p.gthread[q]; }
  const int count = end - first;
  if (algo == 2) {
    // HighwayHash-256: two threads per stream, exactly the half-state code of the fused kernel
    const int s = first + (local >> 1), h = local & 1;
    const bool live = local >= 0 && (local >> 1) < count;
    const WholeStream ws = whole_stream(p, live ? s : first);
    const uint8_t* d = p.data + ws.off;
    HHHalf hs;
    hh_init(hs, p.key, h);
    const int64_t npk = ws.len >> 5;
    const int rem = static_cast<int>(ws.len & 31);
    if (live) {
      for (int64_t q = 0; q < npk; q++) {
        const uint4 v = *reinterpret_cast<const uint4*>(d + q * 32 + 16 * h);
        hh_update(hs, pack64(v.x, v.y), pack64(v.z, v.w));
      }
      if (rem) {
        const uint8_t* tail = d + npk * 32;
        hh_remainder(hs, h, rem, [&](int idx) -> uint32_t { return tail[idx]; });
      }
    }
    uint64_t d0, d1;
    hh_finalize(hs, d0, d1);
    if (live) {
      uint64_t* o = reinterpret_cast<uint64_t*>(p.out + static_cast<int64_t>(s) * 64 + 16 * h);
      o[0] = d0; o[1] = d1;
    }
    return;
  }
  if (local < 0 || local >= count) return;
  const int s = first + local;
  const WholeStream ws = whole_stream(p, s);
  const uint8_t* d = p.data + ws.off;
  const int64_t len = ws.len;
  uint8_t* o = p.out + static_cast<int64_t>(s) * 64;
  if (algo == 1) {
    uint32_t h[8] = {0x6a09e667, 0xbb67ae85, 0x3c6ef372, 0xa54ff53a, 0x510e527f, 0x9b05688c, 0x1f83d9ab, 0x5be0cd19};
    uint32_t w[16];
    const int64_t nfull = len >> 6;
    for (int64_t b = 0; b < nfull; b++) {
#pragma unroll
      for (int q = 0; q < 4; q++) {
        const uint4 v = *reinterpret_cast<const uint4*>(d + b * 64 + q * 16);
        w[4 * q] = bswap32(v.x); w[4 * q + 1] = bswap32(v.y); w[4 * q + 2] = bswap32(v.z); w[4 * q + 3] = bswap32(v.w);
      }
      sha256_compress(h, w);
    }
    // padding: 0x80, zeros, 64-bit big-endian bit length
    const int r = static_cast<int>(len & 63);
    uint8_t blk[128];
    for (int i = 0; i < 128; i++) blk[i] = 0;
    for (int i = 0; i < r; i++) blk[i] = d[nfull * 64 + i];
    blk[r] = 0x80;
    const int total = r < 56 ? 64 : 128;
    const uint64_t bits = static_cast<uint64_t>(len) * 8;
    for (int i = 0; i < 8; i++) blk[total - 1 - i] = static_cast<uint8_t>(bits >> (8 * i));
    for (int bb = 0; bb < total; bb += 64) {
      for (int q = 0; q < 16; q++)
        w[q] = (static_cast<uint32_t>(blk[bb + 4 * q]) << 24) | (static_cast<uint32_t>(blk[bb + 4 * q + 1]) << 16) |
               (static_cast<uint32_t>(blk[bb + 4 * q + 2]) << 8) | blk[bb + 4 * q + 3];
      sha256_compress(h, w);
    }
    for (int i = 0; i < 8; i++) {
      o[4 * i] = static_cast<uint8_t>(h[i] >> 24); o[4 * i + 1] = static_cast<uint8_t>(h[i] >> 16);
      o[4 * i + 2] = static_cast<uint8_t>(h[i] >> 8); o[4 * i + 3] = static_cast<uint8_t>(h[i]);
    }
  } else {  // BLAKE2b-512
    uint64_t h[8];
    for (int i = 0; i < 8; i++) h[i] = kB2IV[i];
    h[0] ^= 0x01010000ull ^ 64;
    uint64_t m[16];
    // all blocks but the last are full 128-byte blocks; the last block (1..128 bytes, or the empty message) is final
    const int64_t nblk = len == 0 ? 1 : (len + 127) / 128;
    for (int64_t b = 0; b < nblk; b++) {
      const bool last = b == nblk - 1;
      const int64_t have = last ? len - b * 128 : 128;
      if (have == 128) {
#pragma unroll
        for (int q = 0; q < 8; q++) {
          const uint4 v = *reinterpret_cast<const uint4*>(d + b * 128 + q * 16);
          m[2 * q] = pack64(v.x, v.y); m[2 * q + 1] = pack64(v.z, v.w);
        }
      } else {
        for (int q = 0; q < 16; q++) {
          uint64_t x = 0;
          for (int i = 0; i < 8; i++) {
            const int64_t pos = q * 8 + i;
            if (pos < have) x |= static_cast<uint64_t>(d[b * 128 + pos]) << (8 * i);
          }
          m[q] = x;
        }
      }
      blake2b_compress(h, m, static_cast<uint64_t>(b * 128 + have), last);
    }
    for (int i = 0; i < 8; i++)
      for (int b = 0; b < 8; b++) o[8 * i + b] = static_cast<uint8_t>(h[i] >> (8 * b));
  }
}

}  // namespace mec
