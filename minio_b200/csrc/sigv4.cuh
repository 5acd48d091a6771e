// sigv4.cuh — the per-chunk signatures of AWS Signature V4 streaming payloads (x-amz-content-sha256:
// STREAMING-AWS4-HMAC-SHA256-PAYLOAD[-TRAILER]), as s3ChunkedReader checks them (cmd/streaming-signature-v4.go:54-94).
//
// Chunk i's signature is HMAC-SHA256(signing key, string to sign), where the string to sign holds SHA-256(chunk i's payload) and
// the signature of chunk i-1.  That previous signature is printed in clear text in chunk i-1's header, so checking every chunk
// against the signature its predecessor claims gives exactly the serial reader's verdicts (the reader moves its seed forward only
// after a match), and every chunk is an independent chain: one thread per chunk, the launch shape of stream_sums_kernel.
//   payload row:  "AWS4-HMAC-SHA256-PAYLOAD\n" date "\n" scope "\n" prev "\n" hex(SHA-256("")) "\n" hex(SHA-256(payload))
//   trailer row:  "AWS4-HMAC-SHA256-TRAILER\n" date "\n" scope "\n" prev "\n" hex(SHA-256(trailer value))
// The HMAC starts from the chaining states of (key ^ ipad) and (key ^ opad), which the host derives from the 32-byte signing key
// (getSigningKey, cmd/signature-v4.go:141) once per call.  The verdict is an exact comparison of the lowercase hex HMAC with the
// 64 claimed bytes: compareSignatureV4 compares strings, so an uppercase claim fails.
#pragma once
#include <cstring>
#include "obj_hash.cuh"

namespace mec {

constexpr int kSigThreads = 32;     // one warp per CTA, as stream_sums_kernel
constexpr int kSigMaxHead = 256;    // date "\n" scope "\n" of a call
constexpr int kSigMsg = 512;        // longest string to sign with its SHA-256 padding: 25 + 256 + 64 + 1 + 65 + 64 + 9 <= 512
constexpr int32_t kSigPayload = 0, kSigTrailer = 1;  // MEC_SIGV4_PAYLOAD / MEC_SIGV4_TRAILER

struct SigRow {
  const uint8_t* msg;  // device: the chunk payload, or the trailer value with its '\n'; any alignment
  int64_t len;
  int64_t out;         // index of the row's verdict byte
  int32_t kind, pad;
  uint8_t prev[64];    // the previous chunk's claimed signature (the seed signature for the first chunk)
  uint8_t claim[64];   // this chunk's claimed signature
};
// What every row of a call shares: the HMAC chaining states of the signing key (zeroed before the call returns) and the
// "date\nscope\n" part of the strings to sign
struct SigCall {
  uint32_t ipad[8], opad[8];
  int32_t head_len, pad;
  uint8_t head[kSigMaxHead];
};
struct SigParams {
  const SigRow* rows;  // sorted by length descending: a warp hashes similar lengths
  int64_t nrows;
  const SigCall* call;
  uint8_t* verdict;    // 1 = the claimed signature matches, 0 = it does not
};

__device__ __forceinline__ uint8_t sig_hex_digit(uint32_t v) { return static_cast<uint8_t>(v < 10 ? '0' + v : 'a' + v - 10); }

__global__ void __launch_bounds__(kSigThreads) sigv4_chunk_kernel(const SigParams p) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * kSigThreads + threadIdx.x;
  if (i >= p.nrows) return;
  const SigRow* r = p.rows + i;
  const SigCall* cl = p.call;
  const int64_t len = r->len;
  const bool payload = r->kind == kSigPayload;
  SumState<2> dg;
  dg.init();
  sum_message(dg, r->msg, len, r->msg + len, 0);

  // the string to sign, then its SHA-256 padding for a message that follows the 64-byte ipad block
  alignas(16) uint8_t m[kSigMsg];
  const char* alg = payload ? "AWS4-HMAC-SHA256-PAYLOAD\n" : "AWS4-HMAC-SHA256-TRAILER\n";
  int n = 0;
  for (int j = 0; j < 25; j++) m[n++] = static_cast<uint8_t>(alg[j]);
  const int hl = cl->head_len;
  for (int j = 0; j < hl; j++) m[n++] = cl->head[j];
  for (int j = 0; j < 64; j++) m[n++] = r->prev[j];
  m[n++] = '\n';
  if (payload) {
    const char* empty = "e3b0c44298fc1c149afbf4c8996fb92427ae41e4649b934ca495991b7852b855\n";  // emptySHA256
    for (int j = 0; j < 65; j++) m[n++] = static_cast<uint8_t>(empty[j]);
  }
#pragma unroll
  for (int q = 0; q < 8; q++)
#pragma unroll
    for (int t = 0; t < 8; t++) m[n + 8 * q + t] = sig_hex_digit((dg.h[q] >> (28 - 4 * t)) & 15);
  n += 64;
  const int nb = (n + 9 + 63) >> 6;
  m[n] = 0x80;
  for (int j = n + 1; j < nb * 64 - 8; j++) m[j] = 0;
  const uint64_t bits = static_cast<uint64_t>(64 + n) * 8;
#pragma unroll
  for (int t = 0; t < 8; t++) m[nb * 64 - 8 + t] = static_cast<uint8_t>(bits >> (56 - 8 * t));

  uint32_t h[8], w[16];
#pragma unroll
  for (int j = 0; j < 8; j++) h[j] = cl->ipad[j];
  for (int b = 0; b < nb; b++) {
    const uint32_t* mw = reinterpret_cast<const uint32_t*>(m + 64 * b);
#pragma unroll
    for (int j = 0; j < 16; j++) w[j] = bswap32(mw[j]);
    sha256_compress(h, w);
  }
  // outer hash: the 32-byte inner digest after the opad block
#pragma unroll
  for (int j = 0; j < 8; j++) { w[j] = h[j]; h[j] = cl->opad[j]; }
  w[8] = 0x80000000u;
#pragma unroll
  for (int j = 9; j < 15; j++) w[j] = 0;
  w[15] = (64 + 32) * 8;
  sha256_compress(h, w);

  bool ok = true;
#pragma unroll
  for (int q = 0; q < 8; q++)
#pragma unroll
    for (int t = 0; t < 8; t++) ok &= r->claim[8 * q + t] == sig_hex_digit((h[q] >> (28 - 4 * t)) & 15);
  p.verdict[r->out] = ok ? 1 : 0;
}

// ---- host: the HMAC-SHA256 chaining states of a 32-byte key (FIPS 180-4 compression, RFC 2104 pads) ----------------------------
inline void sig_host_compress(uint32_t (&h)[8], const uint8_t* blk) {
  static const uint32_t K[64] = {
      0x428a2f98, 0x71374491, 0xb5c0fbcf, 0xe9b5dba5, 0x3956c25b, 0x59f111f1, 0x923f82a4, 0xab1c5ed5, 0xd807aa98, 0x12835b01, 0x243185be,
      0x550c7dc3, 0x72be5d74, 0x80deb1fe, 0x9bdc06a7, 0xc19bf174, 0xe49b69c1, 0xefbe4786, 0x0fc19dc6, 0x240ca1cc, 0x2de92c6f, 0x4a7484aa,
      0x5cb0a9dc, 0x76f988da, 0x983e5152, 0xa831c66d, 0xb00327c8, 0xbf597fc7, 0xc6e00bf3, 0xd5a79147, 0x06ca6351, 0x14292967, 0x27b70a85,
      0x2e1b2138, 0x4d2c6dfc, 0x53380d13, 0x650a7354, 0x766a0abb, 0x81c2c92e, 0x92722c85, 0xa2bfe8a1, 0xa81a664b, 0xc24b8b70, 0xc76c51a3,
      0xd192e819, 0xd6990624, 0xf40e3585, 0x106aa070, 0x19a4c116, 0x1e376c08, 0x2748774c, 0x34b0bcb5, 0x391c0cb3, 0x4ed8aa4a, 0x5b9cca4f,
      0x682e6ff3, 0x748f82ee, 0x78a5636f, 0x84c87814, 0x8cc70208, 0x90befffa, 0xa4506ceb, 0xbef9a3f7, 0xc67178f2};
  auto ror = [](uint32_t x, int s) { return (x >> s) | (x << (32 - s)); };
  uint32_t w[64];
  for (int j = 0; j < 16; j++)
    w[j] = (uint32_t(blk[4 * j]) << 24) | (uint32_t(blk[4 * j + 1]) << 16) | (uint32_t(blk[4 * j + 2]) << 8) | blk[4 * j + 3];
  for (int j = 16; j < 64; j++) {
    const uint32_t s0 = ror(w[j - 15], 7) ^ ror(w[j - 15], 18) ^ (w[j - 15] >> 3);
    const uint32_t s1 = ror(w[j - 2], 17) ^ ror(w[j - 2], 19) ^ (w[j - 2] >> 10);
    w[j] = w[j - 16] + s0 + w[j - 7] + s1;
  }
  uint32_t a = h[0], b = h[1], c = h[2], d = h[3], e = h[4], f = h[5], g = h[6], hh = h[7];
  for (int j = 0; j < 64; j++) {
    const uint32_t t1 = hh + (ror(e, 6) ^ ror(e, 11) ^ ror(e, 25)) + ((e & f) ^ (~e & g)) + K[j] + w[j];
    const uint32_t t2 = (ror(a, 2) ^ ror(a, 13) ^ ror(a, 22)) + ((a & b) ^ (a & c) ^ (b & c));
    hh = g; g = f; f = e; e = d + t1; d = c; c = b; b = a; a = t1 + t2;
  }
  h[0] += a; h[1] += b; h[2] += c; h[3] += d; h[4] += e; h[5] += f; h[6] += g; h[7] += hh;
  explicit_bzero(w, sizeof(w));
}

// ipad / opad states of `key` (32 bytes, shorter than the SHA-256 block: zero-padded, not hashed)
inline void sig_key_states(const uint8_t* key, SigCall* call) {
  static const uint32_t iv[8] = {0x6a09e667, 0xbb67ae85, 0x3c6ef372, 0xa54ff53a, 0x510e527f, 0x9b05688c, 0x1f83d9ab, 0x5be0cd19};
  uint8_t blk[64];
  for (int pass = 0; pass < 2; pass++) {
    uint32_t* h = pass ? call->opad : call->ipad;
    const uint8_t x = pass ? 0x5c : 0x36;
    for (int j = 0; j < 64; j++) blk[j] = static_cast<uint8_t>((j < 32 ? key[j] : 0) ^ x);
    uint32_t s[8];
    for (int j = 0; j < 8; j++) s[j] = iv[j];
    sig_host_compress(s, blk);
    for (int j = 0; j < 8; j++) h[j] = s[j];
    explicit_bzero(s, sizeof(s));
  }
  explicit_bzero(blk, sizeof(blk));
}

}  // namespace mec
