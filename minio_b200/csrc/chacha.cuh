// chacha.cuh — DARE 2.0 (minio/sio) ChaCha20-Poly1305 packages sealed and opened on the device (cipher 1 of the header).
//
// The package layout, nonce (header[4:16], bytes 8..11 XORed with the sequence number) and additional data (header[0:4]) are the
// AES packages' (dare.cuh); only the AEAD is RFC 8439 §2.8.  ChaCha20 block 0 under the package nonce gives the Poly1305 key, the
// payload is XORed with blocks 1, 2, ...  The key is the stream's DareStreamKeys::rk[0..7] (big-endian words of the raw key, which
// the AES schedule only appends to).
//
// One CTA of kDareThreads per package row, driven by the DarePkg table of the AES kernel.  Thread t makes ChaCha20 blocks t, t + 256,
// ... of the payload.  The MAC is split as dare_kernel splits GHASH: Poly1305 block i (the additional-data block, the ciphertext
// blocks, the length block) goes to thread i mod 256, which runs Horner with r^256 and aligns its sum with one multiplication by r^e
// (1 <= e <= 256); the partial sums are added mod 2^130 - 5.  r^1..r^256 are built per package in shared memory by an eight-step
// doubling ladder.  A seal writes the ciphertext first and MACs it back from the output; an open checks header and tag before it
// writes any plaintext.
#pragma once
#include <cstdint>

#include "dare.cuh"

namespace mec {

__host__ __device__ __forceinline__ uint32_t chacha_rotl(uint32_t x, int n) {
#ifdef __CUDA_ARCH__
  return __funnelshift_l(x, x, n);
#else
  return (x << n) | (x >> (32 - n));
#endif
}

#define MEC_CHACHA_QR(a, b, c, d)                  \
  a += b; d ^= a; d = chacha_rotl(d, 16);          \
  c += d; b ^= c; b = chacha_rotl(b, 12);          \
  a += b; d ^= a; d = chacha_rotl(d, 8);           \
  c += d; b ^= c; b = chacha_rotl(b, 7);

// The ChaCha20 block function (RFC 8439 §2.3): key and nonce as little-endian words; out = the 16 keystream words
__host__ __device__ __forceinline__ void chacha_block(const uint32_t key[8], uint32_t counter, uint32_t n0, uint32_t n1, uint32_t n2,
                                                      uint32_t out[16]) {
  uint32_t x0 = 0x61707865u, x1 = 0x3320646eu, x2 = 0x79622d32u, x3 = 0x6b206574u;
  uint32_t x4 = key[0], x5 = key[1], x6 = key[2], x7 = key[3], x8 = key[4], x9 = key[5], x10 = key[6], x11 = key[7];
  uint32_t x12 = counter, x13 = n0, x14 = n1, x15 = n2;
#pragma unroll 2
  for (int i = 0; i < 10; i++) {
    MEC_CHACHA_QR(x0, x4, x8, x12) MEC_CHACHA_QR(x1, x5, x9, x13) MEC_CHACHA_QR(x2, x6, x10, x14) MEC_CHACHA_QR(x3, x7, x11, x15)
    MEC_CHACHA_QR(x0, x5, x10, x15) MEC_CHACHA_QR(x1, x6, x11, x12) MEC_CHACHA_QR(x2, x7, x8, x13) MEC_CHACHA_QR(x3, x4, x9, x14)
  }
  out[0] = x0 + 0x61707865u; out[1] = x1 + 0x3320646eu; out[2] = x2 + 0x79622d32u; out[3] = x3 + 0x6b206574u;
  out[4] = x4 + key[0]; out[5] = x5 + key[1]; out[6] = x6 + key[2]; out[7] = x7 + key[3];
  out[8] = x8 + key[4]; out[9] = x9 + key[5]; out[10] = x10 + key[6]; out[11] = x11 + key[7];
  out[12] = x12 + counter; out[13] = x13 + n0; out[14] = x14 + n1; out[15] = x15 + n2;
}
#undef MEC_CHACHA_QR

// An element of GF(2^130 - 5) as five 26-bit limbs, least significant first.  mul and add take limbs below 2^28 and leave limb 1
// below 2^26 + 2^13 and the others below 2^26.  p1305_finish reduces fully.
struct P1305 {
  uint32_t l[5];
};
constexpr uint32_t kP1305Mask = 0x3ffffff;

// 16 bytes as four little-endian words, plus hibit * 2^128
__host__ __device__ __forceinline__ P1305 p1305_from_words(const uint32_t w[4], uint32_t hibit) {
  P1305 a;
  a.l[0] = w[0] & kP1305Mask;
  a.l[1] = ((w[0] >> 26) | (w[1] << 6)) & kP1305Mask;
  a.l[2] = ((w[1] >> 20) | (w[2] << 12)) & kP1305Mask;
  a.l[3] = ((w[2] >> 14) | (w[3] << 18)) & kP1305Mask;
  a.l[4] = (w[3] >> 8) | (hibit << 24);
  return a;
}

// the carry chain shared by mul and add: d[i] < 2^62 in, limbs as documented at P1305 out
__host__ __device__ __forceinline__ P1305 p1305_carry(uint64_t d0, uint64_t d1, uint64_t d2, uint64_t d3, uint64_t d4) {
  P1305 r;
  d1 += d0 >> 26; r.l[0] = static_cast<uint32_t>(d0) & kP1305Mask;
  d2 += d1 >> 26; r.l[1] = static_cast<uint32_t>(d1) & kP1305Mask;
  d3 += d2 >> 26; r.l[2] = static_cast<uint32_t>(d2) & kP1305Mask;
  d4 += d3 >> 26; r.l[3] = static_cast<uint32_t>(d3) & kP1305Mask;
  r.l[4] = static_cast<uint32_t>(d4) & kP1305Mask;
  const uint64_t t = r.l[0] + (d4 >> 26) * 5;  // 2^130 = 5 mod p
  r.l[0] = static_cast<uint32_t>(t) & kP1305Mask;
  r.l[1] += static_cast<uint32_t>(t >> 26);
  return r;
}

__host__ __device__ __forceinline__ P1305 p1305_mul(const P1305& a, const P1305& b) {
  const uint64_t a0 = a.l[0], a1 = a.l[1], a2 = a.l[2], a3 = a.l[3], a4 = a.l[4];
  const uint64_t b0 = b.l[0], b1 = b.l[1], b2 = b.l[2], b3 = b.l[3], b4 = b.l[4];
  const uint64_t s1 = b1 * 5, s2 = b2 * 5, s3 = b3 * 5, s4 = b4 * 5;
  return p1305_carry(a0 * b0 + a1 * s4 + a2 * s3 + a3 * s2 + a4 * s1,
                     a0 * b1 + a1 * b0 + a2 * s4 + a3 * s3 + a4 * s2,
                     a0 * b2 + a1 * b1 + a2 * b0 + a3 * s4 + a4 * s3,
                     a0 * b3 + a1 * b2 + a2 * b1 + a3 * b0 + a4 * s4,
                     a0 * b4 + a1 * b3 + a2 * b2 + a3 * b1 + a4 * b0);
}

__host__ __device__ __forceinline__ P1305 p1305_add(const P1305& a, const P1305& b) {
  return p1305_carry(uint64_t{a.l[0]} + b.l[0], uint64_t{a.l[1]} + b.l[1], uint64_t{a.l[2]} + b.l[2], uint64_t{a.l[3]} + b.l[3],
                     uint64_t{a.l[4]} + b.l[4]);
}

// (a mod p + s) mod 2^128 as four little-endian words: the tag.  a's limbs below 2^31.
__host__ __device__ __forceinline__ void p1305_finish(const P1305& a, const uint32_t s[4], uint32_t tag[4]) {
  uint32_t h0 = a.l[0], h1 = a.l[1], h2 = a.l[2], h3 = a.l[3], h4 = a.l[4], c;
  // to 26-bit limbs of a value below 2^130 + 2^8 (limb 4 reaches 2^26 only at or above 2^130, where g below is taken)
  c = h0 >> 26; h0 &= kP1305Mask; h1 += c;
  c = h1 >> 26; h1 &= kP1305Mask; h2 += c;
  c = h2 >> 26; h2 &= kP1305Mask; h3 += c;
  c = h3 >> 26; h3 &= kP1305Mask; h4 += c;
  c = h4 >> 26; h4 &= kP1305Mask; h0 += c * 5;
  c = h0 >> 26; h0 &= kP1305Mask; h1 += c;
  c = h1 >> 26; h1 &= kP1305Mask; h2 += c;
  c = h2 >> 26; h2 &= kP1305Mask; h3 += c;
  c = h3 >> 26; h3 &= kP1305Mask; h4 += c;
  // g = h + 5 - 2^130: h >= p exactly when g does not borrow, and then h mod p = g
  uint32_t g0 = h0 + 5;       c = g0 >> 26; g0 &= kP1305Mask;
  uint32_t g1 = h1 + c;       c = g1 >> 26; g1 &= kP1305Mask;
  uint32_t g2 = h2 + c;       c = g2 >> 26; g2 &= kP1305Mask;
  uint32_t g3 = h3 + c;       c = g3 >> 26; g3 &= kP1305Mask;
  const uint32_t g4 = h4 + c - (1u << 26);
  const uint32_t keep = (g4 >> 31) - 1;  // all ones: take g
  h0 = (h0 & ~keep) | (g0 & keep); h1 = (h1 & ~keep) | (g1 & keep); h2 = (h2 & ~keep) | (g2 & keep);
  h3 = (h3 & ~keep) | (g3 & keep); h4 = (h4 & ~keep) | (g4 & keep);
  const uint32_t f0 = h0 | (h1 << 26), f1 = (h1 >> 6) | (h2 << 20), f2 = (h2 >> 12) | (h3 << 14), f3 = (h3 >> 18) | (h4 << 8);
  uint64_t f = uint64_t{f0} + s[0];
  tag[0] = static_cast<uint32_t>(f);
  f = uint64_t{f1} + s[1] + (f >> 32); tag[1] = static_cast<uint32_t>(f);
  f = uint64_t{f2} + s[2] + (f >> 32); tag[2] = static_cast<uint32_t>(f);
  f = uint64_t{f3} + s[3] + (f >> 32); tag[3] = static_cast<uint32_t>(f);
}

// r of the one-time key words k[0..3], clamped (RFC 8439 §2.5.1)
__host__ __device__ __forceinline__ P1305 p1305_clamp(const uint32_t k[4]) {
  const uint32_t w[4] = {k[0] & 0x0fffffffu, k[1] & 0x0ffffffcu, k[2] & 0x0ffffffcu, k[3] & 0x0ffffffcu};
  return p1305_from_words(w, 0);
}

// 16 bytes at p (n <= 16 valid, the rest zero) as four little-endian words
__device__ __forceinline__ void chacha_load(const uint8_t* p, int n, uint32_t w[4]) {
  if (n == 16 && (reinterpret_cast<uintptr_t>(p) & 15) == 0) {
    const uint4 v = *reinterpret_cast<const uint4*>(p);
    w[0] = v.x; w[1] = v.y; w[2] = v.z; w[3] = v.w;
    return;
  }
  w[0] = w[1] = w[2] = w[3] = 0;
  for (int j = 0; j < n; j++) w[j >> 2] |= uint32_t(p[j]) << (8 * (j & 3));
}
__device__ __forceinline__ void chacha_store(uint8_t* p, int n, const uint32_t w[4]) {
  if (n == 16 && (reinterpret_cast<uintptr_t>(p) & 15) == 0) {
    *reinterpret_cast<uint4*>(p) = make_uint4(w[0], w[1], w[2], w[3]);
    return;
  }
  for (int j = 0; j < n; j++) p[j] = static_cast<uint8_t>(w[j >> 2] >> (8 * (j & 3)));
}

// the open kernel's mark for a row it leaves to dare_kernel: not cipher 1, or a stream that does not open ChaCha20
constexpr uint32_t kChachaSkip = 0xff;

struct ChachaSmem {
  P1305 rp[kDareThreads];        // r^(e+1) of the package's one-time key
  P1305 red[kDareThreads / 32];
  uint32_t key[8];               // the stream's key, little-endian words
  uint32_t nonce[3];             // AEAD nonce, little-endian words
  uint32_t s[4];                 // the second half of the one-time key
  uint8_t hdr[16];
  uint32_t status;
};

// Thread t's ChaCha20 blocks of the payload (counter b + 1 for payload block b): in -> out
__device__ __forceinline__ void chacha_xor(const ChachaSmem& sm, const uint8_t* in, uint8_t* out, int len) {
  const int nch = (len + 63) >> 6;
  for (int b = threadIdx.x; b < nch; b += kDareThreads) {
    uint32_t ks[16];
    chacha_block(sm.key, static_cast<uint32_t>(b + 1), sm.nonce[0], sm.nonce[1], sm.nonce[2], ks);
#pragma unroll
    for (int q = 0; q < 4; q++) {
      const int off = 64 * b + 16 * q, n = min(16, len - off);
      if (n <= 0) break;
      uint32_t w[4];
      chacha_load(in + off, n, w);
      for (int j = 0; j < 4; j++) w[j] ^= ks[4 * q + j];
      chacha_store(out + off, n, w);
    }
  }
}

// kSeal: in = plaintext, out = the package (header 0x20, 1).  Open: launched behind dare_kernel<false> over the same rows; a row
// whose header names cipher 1 and whose stream allows ChaCha20 (DareStreamKeys::nonce[kDarePolicy]) gets its status rewritten and,
// if it authenticates, its plaintext; every other row is left as dare_kernel left it.
template <bool kSeal>
__global__ void __launch_bounds__(kDareThreads, 4) dare_chacha_kernel(const DareStreamKeys* __restrict__ keys, const DarePkg* __restrict__ pkgs,
                                                                  const uint8_t* __restrict__ in, uint8_t* __restrict__ out,
                                                                  uint8_t* __restrict__ status) {
  __shared__ ChachaSmem sm;
  const int t = threadIdx.x;
  const DarePkg row = pkgs[blockIdx.x];
  const DareStreamKeys& K = keys[row.stream];
  const int len = row.len;
  const uint8_t* src = in + row.in_off;
  uint8_t* dst = out + row.out_off;
  if (t < 8) sm.key[t] = dare_bswap(K.rk[t]);
  if (t == 0) {
    uint32_t st = kDareOk;
    if (kSeal) {
      sm.hdr[0] = 0x20; sm.hdr[1] = 1;
      sm.hdr[2] = static_cast<uint8_t>((len - 1) & 0xff); sm.hdr[3] = static_cast<uint8_t>((len - 1) >> 8);
      for (int j = 0; j < 12; j++) sm.hdr[4 + j] = K.nonce[j];
      sm.hdr[4] = row.final ? (sm.hdr[4] | 0x80) : (sm.hdr[4] & 0x7f);
      for (int j = 0; j < 16; j++) dst[j] = sm.hdr[j];
    } else {
      for (int j = 0; j < 16; j++) sm.hdr[j] = src[j];
      if (sm.hdr[0] != 0x20 || sm.hdr[1] != 1 || !K.nonce[kDarePolicy]) st = kChachaSkip;
      else st = dare_check_header(sm.hdr, in + row.ref_off, len, row.final != 0, 1);
    }
    const uint8_t* h = sm.hdr;
    sm.nonce[0] = uint32_t(h[4]) | (uint32_t(h[5]) << 8) | (uint32_t(h[6]) << 16) | (uint32_t(h[7]) << 24);
    sm.nonce[1] = uint32_t(h[8]) | (uint32_t(h[9]) << 8) | (uint32_t(h[10]) << 16) | (uint32_t(h[11]) << 24);
    sm.nonce[2] = (uint32_t(h[12]) | (uint32_t(h[13]) << 8) | (uint32_t(h[14]) << 16) | (uint32_t(h[15]) << 24)) ^ row.seq;
    sm.status = st;
  }
  __syncthreads();
  if (!kSeal && sm.status != kDareOk) {
    if (t == 0 && sm.status != kChachaSkip) status[blockIdx.x] = static_cast<uint8_t>(sm.status);
    return;
  }
  if (t == 0) {  // the one-time key: block 0
    uint32_t k0[16];
    chacha_block(sm.key, 0, sm.nonce[0], sm.nonce[1], sm.nonce[2], k0);
    sm.rp[0] = p1305_clamp(k0);
    for (int j = 0; j < 4; j++) sm.s[j] = k0[4 + j];
  }
  uint8_t* ct_out = dst + 16;
  if (kSeal) chacha_xor(sm, src, ct_out, len);
  __syncthreads();  // r, and (seal) the ciphertext the MAC reads back
  // r^1..r^256: at step j threads t < 2^j make r^(2^j + t + 1) = r^(t + 1) * r^(2^j)
#pragma unroll 1
  for (int j = 0; j < 8; j++) {
    const int p = 1 << j;
    if (t < p) sm.rp[p + t] = p1305_mul(sm.rp[t], sm.rp[p - 1]);
    __syncthreads();
  }
  const uint8_t* ct = kSeal ? ct_out : src + 16;
  const int nblk = (len + 15) >> 4;
  const int T = nblk + 2;  // additional-data block, ciphertext blocks, length block
  P1305 acc = {{0, 0, 0, 0, 0}};
  int last = -1;
  for (int i = t; i < T; i += kDareThreads) {
    uint32_t w[4] = {0, 0, 0, 0};
    if (i == 0) {
      w[0] = uint32_t(sm.hdr[0]) | (uint32_t(sm.hdr[1]) << 8) | (uint32_t(sm.hdr[2]) << 16) | (uint32_t(sm.hdr[3]) << 24);
    } else if (i == T - 1) {
      w[0] = 4; w[2] = static_cast<uint32_t>(len);
    } else {
      const int b = i - 1;
      chacha_load(ct + 16 * b, min(16, len - 16 * b), w);
    }
    if (last >= 0) acc = p1305_mul(acc, sm.rp[kDareThreads - 1]);
    const P1305 c = p1305_from_words(w, 1);
    for (int j = 0; j < 5; j++) acc.l[j] += c.l[j];
    last = i;
  }
  if (last >= 0) acc = p1305_mul(acc, sm.rp[T - last - 1]);
  for (int o = 16; o > 0; o >>= 1) {
    P1305 x;
    for (int j = 0; j < 5; j++) x.l[j] = __shfl_xor_sync(0xffffffffu, acc.l[j], o);
    acc = p1305_add(acc, x);
  }
  if ((t & 31) == 0) sm.red[t >> 5] = acc;
  __syncthreads();
  if (t == 0) {
    P1305 sum = sm.red[0];
    for (int w = 1; w < kDareThreads / 32; w++) sum = p1305_add(sum, sm.red[w]);
    uint32_t tag[4];
    p1305_finish(sum, sm.s, tag);
    if (kSeal) {
      chacha_store(ct_out + len, 16, tag);
    } else {
      uint32_t want[4];
      chacha_load(src + 16 + len, 16, want);
      const uint32_t diff = (want[0] ^ tag[0]) | (want[1] ^ tag[1]) | (want[2] ^ tag[2]) | (want[3] ^ tag[3]);
      sm.status = diff ? kDareNotAuthentic : kDareOk;
      status[blockIdx.x] = static_cast<uint8_t>(sm.status);
    }
  }
  if (kSeal) return;
  __syncthreads();
  if (sm.status != kDareOk) return;  // no plaintext of a package that does not authenticate
  chacha_xor(sm, src + 16, dst, len);
}

}  // namespace mec
