// test_chacha.cu — runs the __host__ __device__ building blocks of chacha.cuh (the ChaCha20 block function and the Poly1305 field
// arithmetic mod 2^130 - 5) ON THE HOST and prints every operand and result, one case per line, for tests/test_dare_chacha_abi.py
// to check against Python integers and tests/chacha_ref.py.  Built by nvcc as a host-only executable (no GPU needed).
//   mul a0..a4 b0..b4 r0..r4       p1305_mul (limbs)
//   add a0..a4 b0..b4 r0..r4       p1305_add
//   fin a0..a4 s0..s3 t0..t3       p1305_finish (the tag words)
//   clamp k0..k3 r0..r4            p1305_clamp
//   blk key0..key7 ctr n0 n1 n2 out0..out15
#include <cstdint>
#include <cstdio>

#include "../../minio_b200/csrc/chacha.cuh"
using namespace mec;

static uint64_t rng_state = 0x9e3779b97f4a7c15ull;
static uint32_t rnd() {
  rng_state ^= rng_state << 13; rng_state ^= rng_state >> 7; rng_state ^= rng_state << 17;
  return static_cast<uint32_t>(rng_state >> 16);
}
static P1305 limbs(uint32_t a, uint32_t b, uint32_t c, uint32_t d, uint32_t e) { return P1305{{a, b, c, d, e}}; }
static P1305 rnd_limbs(uint32_t bound) {  // limbs below bound
  P1305 x;
  for (auto& l : x.l) l = rnd() % bound;
  return x;
}
static void put(const P1305& x) { for (uint32_t l : x.l) printf(" %u", l); }
static void mul(const P1305& a, const P1305& b) { printf("mul"); put(a); put(b); put(p1305_mul(a, b)); printf("\n"); }
static void add(const P1305& a, const P1305& b) { printf("add"); put(a); put(b); put(p1305_add(a, b)); printf("\n"); }
static void fin(const P1305& a, const uint32_t s[4]) {
  uint32_t t[4];
  p1305_finish(a, s, t);
  printf("fin"); put(a);
  for (int i = 0; i < 4; i++) printf(" %u", s[i]);
  for (int i = 0; i < 4; i++) printf(" %u", t[i]);
  printf("\n");
}

int main() {
  const uint32_t M = kP1305Mask, top = (1u << 28) - 1;
  const uint32_t zero[4] = {0, 0, 0, 0}, ones[4] = {~0u, ~0u, ~0u, ~0u};
  // crafted: the largest clamped r, limbs at the input bound (carries out of every limb), p - 1 and 2^130 - 1 as operands
  const uint32_t kmax[4] = {~0u, ~0u, ~0u, ~0u};
  const P1305 rmax = p1305_clamp(kmax);
  printf("clamp %u %u %u %u", kmax[0], kmax[1], kmax[2], kmax[3]); put(rmax); printf("\n");
  const P1305 big = limbs(top, top, top, top, top), pm1 = limbs(M - 5, M, M, M, M), all = limbs(M, M, M, M, M);
  const P1305 after = limbs(M, M + (1u << 13) - 1, M, M, M);  // the largest mul / add output
  for (const P1305& a : {big, pm1, all, after, rmax})
    for (const P1305& b : {big, pm1, all, after, rmax}) { mul(a, b); add(a, b); }
  // crafted finals: p - 1, p, p + 1, 2^130 - 1 and non-canonical forms around them, with s = 0 and s = 2^128 - 1
  const P1305 finals[] = {pm1, limbs(M - 4, M, M, M, M), limbs(M - 3, M, M, M, M), all, limbs(0, 0, 0, 0, 0), limbs(5, 0, 0, 0, 0),
                          limbs(M + 1, M, M, M, M), limbs(0, M + 1, M, M, M), limbs(M, M, M, M, M + 1), after,
                          limbs((1u << 31) - 1, (1u << 31) - 1, (1u << 31) - 1, (1u << 31) - 1, (1u << 31) - 1),
                          limbs(M - 4, M, M, M, M + 1), limbs(M - 5, M, M, M, (1u << 26) + M)};
  for (const P1305& a : finals) { fin(a, zero); fin(a, ones); }
  // random: operands up to the input bounds, products fed back as the kernel feeds them, finals of random sums
  for (int i = 0; i < 2000; i++) {
    const P1305 a = rnd_limbs(i & 1 ? 1u << 28 : 1u << 26), b = rnd_limbs(i & 2 ? 1u << 28 : 1u << 26);
    mul(a, b);
    add(a, b);
    P1305 x = p1305_mul(a, b);
    for (int j = 0; j < 3; j++) x = p1305_mul(p1305_add(x, a), b);
    const uint32_t s[4] = {rnd(), rnd(), rnd(), rnd()};
    fin(x, s);
    fin(rnd_limbs(1u << 31), s);
    const uint32_t k[4] = {rnd(), rnd(), rnd(), rnd()};
    printf("clamp %u %u %u %u", k[0], k[1], k[2], k[3]); put(p1305_clamp(k)); printf("\n");
  }
  // the block function: RFC 8439 §2.3.2's inputs, then random keys, counters and nonces
  for (int i = 0; i < 200; i++) {
    uint32_t key[8], n[3], ctr, out[16];
    if (i == 0) {
      for (int j = 0; j < 8; j++) key[j] = (4u * j) | ((4u * j + 1) << 8) | ((4u * j + 2) << 16) | ((4u * j + 3) << 24);
      n[0] = 0x09000000u; n[1] = 0x4a000000u; n[2] = 0; ctr = 1;
    } else {
      for (auto& w : key) w = rnd();
      for (auto& w : n) w = rnd();
      ctr = i < 100 ? static_cast<uint32_t>(i) : rnd();
    }
    chacha_block(key, ctr, n[0], n[1], n[2], out);
    printf("blk");
    for (uint32_t w : key) printf(" %u", w);
    printf(" %u %u %u %u", ctr, n[0], n[1], n[2]);
    for (uint32_t w : out) printf(" %u", w);
    printf("\n");
  }
  printf("done\n");
  return 0;
}
