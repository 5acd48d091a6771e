// dare.cuh — DARE 2.0 (minio/sio) AES-256-GCM packages sealed and opened on the device.
//
// Package layout in include/minio_ec.h.  GCM: CTR from counter 2 (J0 = nonce | 1 masks the tag), GHASH over the additional-data
// block, the ciphertext blocks and the length block.  One CTA per package, driven by a table of DarePkg rows (any number of streams
// and keys per launch).  Thread t runs AES on GHASH blocks t, t + 256, ... and a Horner run over them with H^256, aligned by one
// multiplication with H^e (1 <= e <= 256); the runs are XORed together.  dare_setup_kernel expands the key schedule and computes
// H = E_K(0) and H^1..H^256 per stream from the raw key, dare_tables_kernel the AES tables once per codec.  Open checks header,
// final bit, nonce and tag before any plaintext.  Packages that name ChaCha20-Poly1305 (cipher 1) are chacha.cuh's.
#pragma once
#include <cstdint>

namespace mec {

constexpr int kDarePkg = 65536;                 // payload bytes of a full package
constexpr int kDareOverhead = 32;               // header + tag
constexpr int kDareEPkg = kDarePkg + kDareOverhead;
constexpr int kDareThreads = 256;

enum : uint8_t { kDareOk = 0, kDareNotAuthentic = 1, kDareUnsupported = 2 };

struct DarePkg {
  int64_t in_off;   // seal: plaintext; open: the package (header first)
  int64_t out_off;  // seal: where the package goes; open: where its plaintext goes
  int64_t ref_off;  // open: the in offset of a package whose nonce is the stream's (the first one of the stream in this call)
  int32_t len;      // payload bytes, 1..65536
  uint32_t seq;     // sequence number
  int32_t stream;   // key, H powers and (seal) nonce of this stream
  int32_t final;    // the part's last package
};

// The host writes the first kDareKeyHead bytes of a stream (nonce, policy byte and the raw key as rk[0..7]); dare_setup_kernel the rest.
struct DareStreamKeys {
  uint8_t nonce[16];     // seal: the stream's 12 nonce bytes; nonce[kDarePolicy]: the stream opens ChaCha20-Poly1305 packages
  uint32_t rk[60];       // AES-256 key schedule, big-endian words
  uint64_t hpow[256][2]; // H^(e+1) as (hi, lo) big-endian halves
};
constexpr size_t kDareKeyHead = 16 + 32;
constexpr int kDarePolicy = 12;

// The header checks of an open, in order: version, cipher, length against the position, final bit, the stream's nonce (ref: the
// header of the stream's first package in the call).  `cipher` is the AEAD the caller opens (0 AES-256-GCM, 1 ChaCha20-Poly1305); a
// package that names the other one is kDareUnsupported, as is DARE 1.0.
__device__ __forceinline__ uint32_t dare_check_header(const uint8_t* hdr, const uint8_t* ref, int len, bool final, uint8_t cipher) {
  uint32_t st = kDareOk;
  if (hdr[0] != 0x20) st = hdr[0] == 0x10 ? kDareUnsupported : kDareNotAuthentic;
  else if (hdr[1] != cipher) st = hdr[1] <= 1 ? kDareUnsupported : kDareNotAuthentic;
  else if ((hdr[2] | (hdr[3] << 8)) + 1 != len) st = kDareNotAuthentic;
  else if (((hdr[4] & 0x80) != 0) != final) st = kDareNotAuthentic;
  else {
    if (((hdr[4] ^ ref[4]) & 0x7f) != 0) st = kDareNotAuthentic;
    for (int j = 5; j < 16; j++) if (hdr[j] != ref[j]) st = kDareNotAuthentic;
  }
  return st;
}

struct DareTables {
  uint32_t te[4][256];
  uint32_t sbox[256];
};

__host__ __device__ inline uint8_t dare_gmul8(uint8_t a, uint8_t b) {
  uint8_t p = 0;
  for (int i = 0; i < 8; i++) {
    if (b & 1) p ^= a;
    const uint8_t hi = a & 0x80;
    a = static_cast<uint8_t>(a << 1);
    if (hi) a ^= 0x1b;
    b >>= 1;
  }
  return p;
}
// the AES S-box: multiplicative inverse in GF(2^8) followed by the affine map
__host__ __device__ inline uint8_t dare_sbox(uint8_t x) {
  uint8_t inv = 0;
  if (x) {  // x^254
    uint8_t r = 1, b = x;
    for (int e = 254; e; e >>= 1) {
      if (e & 1) r = dare_gmul8(r, b);
      b = dare_gmul8(b, b);
    }
    inv = r;
  }
  uint8_t s = inv;
  for (int i = 1; i <= 4; i++) s ^= static_cast<uint8_t>((inv << i) | (inv >> (8 - i)));
  return s ^ 0x63;
}

// Te0[x] = (2s, s, s, 3s) big-endian; Te1..Te3 are its byte rotations
__global__ void dare_tables_kernel(DareTables* t) {
  const int x = threadIdx.x;
  const uint8_t s = dare_sbox(static_cast<uint8_t>(x));
  const uint32_t w = (uint32_t(dare_gmul8(s, 2)) << 24) | (uint32_t(s) << 16) | (uint32_t(s) << 8) | dare_gmul8(s, 3);
  t->te[0][x] = w;
  t->te[1][x] = (w >> 8) | (w << 24);
  t->te[2][x] = (w >> 16) | (w << 16);
  t->te[3][x] = (w >> 24) | (w << 8);
  t->sbox[x] = s;
}

struct DareSmem {
  uint32_t te[4][256];
  uint32_t sbox[256];
  uint32_t rk[60];
  uint64_t mh[16], ml[16];  // 4-bit table of H^256
  uint64_t r4[16];          // dare_last4
  uint64_t red[kDareThreads / 32][2];
  uint32_t nonce[3];        // AEAD nonce as big-endian words
  uint8_t hdr[16];
  uint32_t status;
};

__host__ __device__ __forceinline__ void dare_aes(const DareSmem& sm, uint32_t s0, uint32_t s1, uint32_t s2, uint32_t s3, uint32_t out[4]) {
  const uint32_t* rk = sm.rk;
  s0 ^= rk[0]; s1 ^= rk[1]; s2 ^= rk[2]; s3 ^= rk[3];
#pragma unroll
  for (int r = 1; r < 14; r++) {
    const uint32_t t0 = sm.te[0][s0 >> 24] ^ sm.te[1][(s1 >> 16) & 0xff] ^ sm.te[2][(s2 >> 8) & 0xff] ^ sm.te[3][s3 & 0xff] ^ rk[4 * r];
    const uint32_t t1 = sm.te[0][s1 >> 24] ^ sm.te[1][(s2 >> 16) & 0xff] ^ sm.te[2][(s3 >> 8) & 0xff] ^ sm.te[3][s0 & 0xff] ^ rk[4 * r + 1];
    const uint32_t t2 = sm.te[0][s2 >> 24] ^ sm.te[1][(s3 >> 16) & 0xff] ^ sm.te[2][(s0 >> 8) & 0xff] ^ sm.te[3][s1 & 0xff] ^ rk[4 * r + 2];
    const uint32_t t3 = sm.te[0][s3 >> 24] ^ sm.te[1][(s0 >> 16) & 0xff] ^ sm.te[2][(s1 >> 8) & 0xff] ^ sm.te[3][s2 & 0xff] ^ rk[4 * r + 3];
    s0 = t0; s1 = t1; s2 = t2; s3 = t3;
  }
  const uint32_t* S = sm.sbox;
  out[0] = (S[s0 >> 24] << 24 | S[(s1 >> 16) & 0xff] << 16 | S[(s2 >> 8) & 0xff] << 8 | S[s3 & 0xff]) ^ rk[56];
  out[1] = (S[s1 >> 24] << 24 | S[(s2 >> 16) & 0xff] << 16 | S[(s3 >> 8) & 0xff] << 8 | S[s0 & 0xff]) ^ rk[57];
  out[2] = (S[s2 >> 24] << 24 | S[(s3 >> 16) & 0xff] << 16 | S[(s0 >> 8) & 0xff] << 8 | S[s1 & 0xff]) ^ rk[58];
  out[3] = (S[s3 >> 24] << 24 | S[(s0 >> 16) & 0xff] << 16 | S[(s1 >> 8) & 0xff] << 8 | S[s2 & 0xff]) ^ rk[59];
}

// GF(2^128) product in GCM's bit order (NIST SP 800-38D, Algorithm 1): elements as (hi, lo) big-endian halves
__host__ __device__ __forceinline__ void dare_gfmul(uint64_t xh, uint64_t xl, uint64_t yh, uint64_t yl, uint64_t& zh, uint64_t& zl) {
  uint64_t h = 0, l = 0;
  for (int i = 0; i < 128; i++) {
    const uint64_t bit = i < 64 ? (xh >> (63 - i)) & 1 : (xl >> (127 - i)) & 1;
    const uint64_t m = 0 - bit;
    h ^= yh & m; l ^= yl & m;
    const uint64_t lsb = yl & 1;
    yl = (yl >> 1) | (yh << 63);
    yh = (yh >> 1) ^ ((0 - lsb) & 0xE100000000000000ull);
  }
  zh = h; zl = l;
}

// 4-bit table of a fixed multiplier (Shoup): entry j = j * Y for the nibble j in GCM's bit order
__host__ __device__ __forceinline__ void dare_table4(uint64_t yh, uint64_t yl, uint64_t* th, uint64_t* tl) {
  th[0] = tl[0] = 0;
  th[8] = yh; tl[8] = yl;
  for (int i = 4; i > 0; i >>= 1) {
    const uint64_t lsb = yl & 1;
    yl = (yl >> 1) | (yh << 63);
    yh = (yh >> 1) ^ ((0 - lsb) & 0xE100000000000000ull);
    th[i] = yh; tl[i] = yl;
  }
  for (int i = 2; i <= 8; i *= 2)
    for (int j = 1; j < i; j++) { th[i + j] = th[i] ^ th[j]; tl[i + j] = tl[i] ^ tl[j]; }
}

// reduction of the four bits a nibble shift drops off (x^128 = x^7 + x^2 + x + 1 in GCM's reflected order), at bit 48
__host__ __device__ inline uint64_t dare_last4(int j) {
  constexpr uint16_t kLast4[16] = {0x0000, 0x1c20, 0x3840, 0x2460, 0x7080, 0x6ca0, 0x48c0, 0x54e0,
                                   0xe100, 0xfd20, 0xd940, 0xc560, 0x9180, 0x8da0, 0xa9c0, 0xb5e0};
  return static_cast<uint64_t>(kLast4[j]) << 48;
}

// X *= Y with Y's 4-bit table (th, tl) and the reduction table r4[j] = dare_last4(j)
__host__ __device__ __forceinline__ void dare_mul_table(const uint64_t* th, const uint64_t* tl, const uint64_t* r4, uint64_t& xh, uint64_t& xl) {
  uint64_t zh = 0, zl = 0;
#pragma unroll
  for (int i = 15; i >= 0; i--) {
    const uint32_t byte = static_cast<uint32_t>(i < 8 ? xh >> (8 * (7 - i)) : xl >> (8 * (15 - i))) & 0xff;
#pragma unroll
    for (int half = 0; half < 2; half++) {
      const uint32_t nib = half == 0 ? byte & 0xf : byte >> 4;
      if (!(i == 15 && half == 0)) {
        const uint32_t rem = static_cast<uint32_t>(zl & 0xf);
        zl = (zh << 60) | (zl >> 4);
        zh = (zh >> 4) ^ r4[rem];
      }
      zh ^= th[nib]; zl ^= tl[nib];
    }
  }
  xh = zh; xl = zl;
}

__host__ __device__ __forceinline__ uint32_t dare_bswap(uint32_t x) {
#ifdef __CUDA_ARCH__
  return __byte_perm(x, 0, 0x0123);
#else
  return __builtin_bswap32(x);
#endif
}

// 16 bytes at p (n <= 16 valid, the rest zero) as four big-endian words
__device__ __forceinline__ void dare_load(const uint8_t* p, int n, uint32_t w[4]) {
  if (n == 16 && (reinterpret_cast<uintptr_t>(p) & 15) == 0) {
    const uint4 v = *reinterpret_cast<const uint4*>(p);
    w[0] = dare_bswap(v.x); w[1] = dare_bswap(v.y); w[2] = dare_bswap(v.z); w[3] = dare_bswap(v.w);
    return;
  }
  w[0] = w[1] = w[2] = w[3] = 0;
  for (int j = 0; j < n; j++) w[j >> 2] |= uint32_t(p[j]) << (24 - 8 * (j & 3));
}
__device__ __forceinline__ void dare_store(uint8_t* p, int n, const uint32_t w[4]) {
  if (n == 16 && (reinterpret_cast<uintptr_t>(p) & 15) == 0) {
    *reinterpret_cast<uint4*>(p) = make_uint4(dare_bswap(w[0]), dare_bswap(w[1]), dare_bswap(w[2]), dare_bswap(w[3]));
    return;
  }
  for (int j = 0; j < n; j++) p[j] = static_cast<uint8_t>(w[j >> 2] >> (24 - 8 * (j & 3)));
}

// Per stream (one CTA): the AES-256 key schedule from rk[0..7] (FIPS-197 §5.2), H = E_K(0^128) and H^1..H^256 by a doubling
// ladder: at step j one thread builds the 4-bit table of H^(2^j), then threads t < 2^j make H^(2^j+t+1) = H^(t+1) * H^(2^j).
__global__ void __launch_bounds__(kDareThreads) dare_setup_kernel(const DareTables* __restrict__ tabs, DareStreamKeys* keys) {
  __shared__ DareSmem sm;
  __shared__ uint64_t hp[256][2];
  DareStreamKeys& K = keys[blockIdx.x];
  const int t = threadIdx.x;
  for (int i = t; i < 1024; i += kDareThreads) (&sm.te[0][0])[i] = (&tabs->te[0][0])[i];
  sm.sbox[t] = tabs->sbox[t];
  if (t < 8) sm.rk[t] = K.rk[t];
  if (t < 16) sm.r4[t] = dare_last4(t);
  __syncthreads();
  if (t == 0) {
    const uint32_t* S = sm.sbox;
    uint32_t rcon = 1;
    for (int i = 8; i < 60; i++) {
      uint32_t w = sm.rk[i - 1];
      if (i % 8 == 0) {
        w = (w << 8) | (w >> 24);
        w = (S[w >> 24] << 24) | (S[(w >> 16) & 0xff] << 16) | (S[(w >> 8) & 0xff] << 8) | S[w & 0xff];
        w ^= rcon << 24;
        rcon = dare_gmul8(static_cast<uint8_t>(rcon), 2);
      } else if (i % 8 == 4) {
        w = (S[w >> 24] << 24) | (S[(w >> 16) & 0xff] << 16) | (S[(w >> 8) & 0xff] << 8) | S[w & 0xff];
      }
      sm.rk[i] = sm.rk[i - 8] ^ w;
    }
    uint32_t h[4];
    dare_aes(sm, 0, 0, 0, 0, h);
    hp[0][0] = (uint64_t(h[0]) << 32) | h[1];
    hp[0][1] = (uint64_t(h[2]) << 32) | h[3];
  }
  __syncthreads();
  if (t >= 8 && t < 60) K.rk[t] = sm.rk[t];
#pragma unroll 1
  for (int j = 0; j < 8; j++) {
    const int p = 1 << j;  // hp[p - 1] = H^p
    if (t == 0) dare_table4(hp[p - 1][0], hp[p - 1][1], sm.mh, sm.ml);
    __syncthreads();
    if (t < p) {
      uint64_t xh = hp[t][0], xl = hp[t][1];
      dare_mul_table(sm.mh, sm.ml, sm.r4, xh, xl);
      hp[p + t][0] = xh; hp[p + t][1] = xl;
    }
    __syncthreads();
  }
  K.hpow[t][0] = hp[t][0];
  K.hpow[t][1] = hp[t][1];
}

// kSeal: in = plaintext, out = the package.  Open: in = the package, out = plaintext; status[row] = kDare*.
template <bool kSeal>
__global__ void __launch_bounds__(kDareThreads, 4) dare_kernel(const DareTables* __restrict__ tabs, const DareStreamKeys* __restrict__ keys,
                                                          const DarePkg* __restrict__ pkgs, const uint8_t* __restrict__ in,
                                                          uint8_t* __restrict__ out, uint8_t* __restrict__ status) {
  __shared__ DareSmem sm;
  const int t = threadIdx.x;
  const DarePkg row = pkgs[blockIdx.x];
  const DareStreamKeys& K = keys[row.stream];
  for (int i = t; i < 1024; i += kDareThreads) (&sm.te[0][0])[i] = (&tabs->te[0][0])[i];
  sm.sbox[t] = tabs->sbox[t];
  if (t < 60) sm.rk[t] = K.rk[t];
  if (t < 16) sm.r4[t] = dare_last4(t);
  const int len = row.len;
  const uint8_t* src = in + row.in_off;
  uint8_t* dst = out + row.out_off;
  if (t == 0) {
    uint32_t st = kDareOk;
    if (kSeal) {
      sm.hdr[0] = 0x20; sm.hdr[1] = 0;
      sm.hdr[2] = static_cast<uint8_t>((len - 1) & 0xff); sm.hdr[3] = static_cast<uint8_t>((len - 1) >> 8);
      for (int j = 0; j < 12; j++) sm.hdr[4 + j] = K.nonce[j];
      sm.hdr[4] = row.final ? (sm.hdr[4] | 0x80) : (sm.hdr[4] & 0x7f);
      for (int j = 0; j < 16; j++) dst[j] = sm.hdr[j];
    } else {
      for (int j = 0; j < 16; j++) sm.hdr[j] = src[j];
      st = dare_check_header(sm.hdr, in + row.ref_off, len, row.final != 0, 0);
    }
    sm.nonce[0] = (uint32_t(sm.hdr[4]) << 24) | (uint32_t(sm.hdr[5]) << 16) | (uint32_t(sm.hdr[6]) << 8) | sm.hdr[7];
    sm.nonce[1] = (uint32_t(sm.hdr[8]) << 24) | (uint32_t(sm.hdr[9]) << 16) | (uint32_t(sm.hdr[10]) << 8) | sm.hdr[11];
    const uint32_t tail = (uint32_t(sm.hdr[12]) | (uint32_t(sm.hdr[13]) << 8) | (uint32_t(sm.hdr[14]) << 16) | (uint32_t(sm.hdr[15]) << 24)) ^ row.seq;
    sm.nonce[2] = dare_bswap(tail);
    sm.status = st;
    dare_table4(K.hpow[255][0], K.hpow[255][1], sm.mh, sm.ml);
  }
  __syncthreads();
  if (!kSeal && sm.status != kDareOk) {
    if (t == 0) status[blockIdx.x] = static_cast<uint8_t>(sm.status);
    return;
  }
  const uint32_t n0 = sm.nonce[0], n1 = sm.nonce[1], n2 = sm.nonce[2];
  const int nblk = (len + 15) >> 4;
  const int T = nblk + 2;  // additional-data block, ciphertext blocks, length block
  const uint8_t* ct = kSeal ? dst + 16 : src + 16;
  // GHASH runs of this thread: blocks i = t, t + 256, ... < T, Horner with H^256
  uint64_t ah = 0, al = 0;
  int last = -1;
  for (int i = t; i < T; i += kDareThreads) {
    uint32_t x[4];
    if (i == 0) {
      x[0] = (uint32_t(sm.hdr[0]) << 24) | (uint32_t(sm.hdr[1]) << 16) | (uint32_t(sm.hdr[2]) << 8) | sm.hdr[3];
      x[1] = x[2] = x[3] = 0;
    } else if (i == T - 1) {
      const uint64_t bits = static_cast<uint64_t>(len) * 8;
      x[0] = 0; x[1] = 32; x[2] = static_cast<uint32_t>(bits >> 32); x[3] = static_cast<uint32_t>(bits);
    } else {
      const int b = i - 1, n = min(16, len - 16 * b);
      if (kSeal) {
        uint32_t ks[4], p[4];
        dare_aes(sm, n0, n1, n2, static_cast<uint32_t>(b + 2), ks);
        dare_load(src + 16 * b, n, p);
        for (int q = 0; q < 4; q++) x[q] = p[q] ^ ks[q];
        if (n < 16) {  // the ciphertext of a short block is its n bytes, zero padded for GHASH
          for (int j = n; j < 16; j++) x[j >> 2] &= ~(0xffu << (24 - 8 * (j & 3)));
        }
        dare_store(dst + 16 + 16 * b, n, x);
      } else {
        dare_load(ct + 16 * b, n, x);
      }
    }
    if (last >= 0) dare_mul_table(sm.mh, sm.ml, sm.r4, ah, al);
    ah ^= (uint64_t(x[0]) << 32) | x[1];
    al ^= (uint64_t(x[2]) << 32) | x[3];
    last = i;
  }
  if (last >= 0) {
    const int e = T - last;  // 1..256
    dare_gfmul(ah, al, K.hpow[e - 1][0], K.hpow[e - 1][1], ah, al);
  }
  for (int o = 16; o > 0; o >>= 1) {
    ah ^= __shfl_xor_sync(0xffffffffu, ah, o);
    al ^= __shfl_xor_sync(0xffffffffu, al, o);
  }
  if ((t & 31) == 0) { sm.red[t >> 5][0] = ah; sm.red[t >> 5][1] = al; }
  __syncthreads();
  if (t == 0) {
    uint64_t sh = 0, sl = 0;
    for (int w = 0; w < kDareThreads / 32; w++) { sh ^= sm.red[w][0]; sl ^= sm.red[w][1]; }
    uint32_t j0[4];
    dare_aes(sm, n0, n1, n2, 1, j0);
    uint32_t tag[4] = {static_cast<uint32_t>(sh >> 32) ^ j0[0], static_cast<uint32_t>(sh) ^ j0[1],
                       static_cast<uint32_t>(sl >> 32) ^ j0[2], static_cast<uint32_t>(sl) ^ j0[3]};
    if (kSeal) {
      dare_store(dst + 16 + len, 16, tag);
    } else {
      uint32_t want[4];
      dare_load(src + 16 + len, 16, want);
      const uint32_t diff = (want[0] ^ tag[0]) | (want[1] ^ tag[1]) | (want[2] ^ tag[2]) | (want[3] ^ tag[3]);
      sm.status = diff ? kDareNotAuthentic : kDareOk;
      status[blockIdx.x] = static_cast<uint8_t>(sm.status);
    }
  }
  if (kSeal) return;
  __syncthreads();
  if (sm.status != kDareOk) return;  // no plaintext of a package that does not authenticate
  for (int b = t; b < nblk; b += kDareThreads) {
    const int n = min(16, len - 16 * b);
    uint32_t ks[4], c[4];
    dare_aes(sm, n0, n1, n2, static_cast<uint32_t>(b + 2), ks);
    dare_load(ct + 16 * b, n, c);
    for (int q = 0; q < 4; q++) c[q] ^= ks[q];
    dare_store(dst + 16 * b, n, c);
  }
}

}  // namespace mec
