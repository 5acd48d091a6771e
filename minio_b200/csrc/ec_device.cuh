// ec_device.cuh — device building blocks of the fused erasure-code + bitrot kernel (sm_90a).
//
//   * packed GF(2^8) arithmetic on 4 bytes per 32-bit register (poly 0x11D — the field of
//     klauspost/reedsolomon, used by cmd/erasure-coding.go:63,85,106,112)
//   * HighwayHash-256 (minio/highwayhash, keyed as cmd/bitrot.go:37,55-58) with TWO threads per
//     hash stream: a thread owns 64-bit lanes {0,1} or {2,3}; the zipper-merge only mixes lanes
//     inside such a pair, so the per-packet update needs no cross-thread traffic at all.  Only the
//     10 finalisation rounds exchange lanes (one shuffle pair per round).
//   * mbarrier / TMA (cp.async.bulk.tensor) wrappers.
#pragma once
#include "rtc_compat.h"
#include "gf256.h"

namespace mec {

#ifndef MEC_HH_VARIANT
#define MEC_HH_VARIANT 0
#endif

// ---------------------------------------------------------------- small helpers
template <class F, int... I>
__host__ __device__ __forceinline__ void static_for_impl(F&& f, std::integer_sequence<int, I...>) {
  (f(std::integral_constant<int, I>{}), ...);
}
template <int N, class F>
__host__ __device__ __forceinline__ void static_for(F&& f) {
  static_for_impl(static_cast<F&&>(f), std::make_integer_sequence<int, N>{});
}

__host__ __device__ __forceinline__ uint32_t prmt(uint32_t a, uint32_t b, uint32_t sel) {
#ifdef __CUDA_ARCH__
  uint32_t d;
  asm("prmt.b32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(sel));
  return d;
#else  // host restatement (tests/cpp/test_gfplan.cu runs the compile-time GF plans on the CPU)
  const uint64_t pool = (static_cast<uint64_t>(b) << 32) | a;
  uint32_t d = 0;
  for (int i = 0; i < 4; i++) {
    const uint32_t s4 = (sel >> (4 * i)) & 0xfu;
    uint32_t byte = static_cast<uint32_t>(pool >> (8 * (s4 & 7u))) & 0xffu;
    if (s4 & 8u) byte = (byte & 0x80u) ? 0xffu : 0u;
    d |= byte << (8 * i);
  }
  return d;
#endif
}

// ---------------------------------------------------------------- packed GF(2^8)
// multiply each of the 4 packed field elements by x (i.e. by 2) modulo x^8+x^4+x^3+x^2+1: PRMT sign-replicate gives
// 0xff per byte whose msb is set, two ANDs and a shift finish it — 3 ALU-pipe ops, FMA pipe almost idle.  (Variants that
// move work to the FMA pipe through IMAD.HI lose to it; tools/ubench.cu measures the two pipes.)
__host__ __device__ __forceinline__ uint32_t gf_xtime4(uint32_t a) {
  const uint32_t m = prmt(a, 0u, 0xba98u);
  return ((a & 0x7f7f7f7fu) << 1) ^ (m & 0x1d1d1d1du);
}

// One Horner step  acc*x ^ x_terms  in 3 ALU-pipe ops + 1 FMA-pipe op: the byte-msb mask comes from PRMT, the
// doubling is a plain 32-bit add whose cross-byte carry-in bit is masked INSIDE the final LOP3
// ((a+a) & 0xfefefefe == (a & 0x7f7f7f7f) << 1), and the reduction mask is folded into the LOP3 that adds the terms.
__host__ __device__ __forceinline__ uint32_t gf_xtime_add4(uint32_t a, uint32_t x_terms) {
  const uint32_t m = prmt(a, 0u, 0xba98u);  // 0xff per byte whose msb is set
  const uint32_t a2 = a + a;
  const uint32_t y = (m & 0x1d1d1d1du) ^ x_terms;
  return (a2 & 0xfefefefeu) ^ y;
}

// Compile-time specialised  out[j] = XOR_t  coef(j,t) (x) in[t]   on packed words.
//
// (1) Horner over the bit planes of the coefficients: out_j = sum_b x^b P_jb with P_jb the XOR of the inputs whose
//     coefficient has bit b set — doublings are paid per OUTPUT word (at most 7), never per input, and a chain starts at
//     the highest plane that has a term at all.
// (2) Plane sums are assembled from "four Russians" XOR combinations of small input groups.
// (3) Subset-sum change of basis.  The systematic Vandermonde matrix of reedsolomon.New is a Lagrange interpolation at
//     the points 0..k+m-1, and addition in GF(2^8) is XOR, so M[r ^ t][c ^ t] = M[r][c] whenever the data columns and
//     the parity rows are both closed under ^t: every aligned 2^L x 2^L block is an XOR-circulant.  With
//     Z = [[1,0],[1,1]]^(x)L (y_i = XOR of x_j over the bit-subsets j of i; Z is its own inverse over GF(2)),
//     Z * circulant * Z is "subset-triangular": only 3^L of its 4^L entries survive and the sums of circulant entries
//     that appear off the full-degree corner have low degree.  RS(12,4): of the 48 eight-bit coefficients 27 remain,
//     three of them eight-bit — 16 doublings instead of 28 and a third of the XOR terms, ~80 ALU ops per 12-word column
//     instead of ~134.  The inputs are transformed with L*2^(L-1) XORs per block, the outputs likewise afterwards.
//     Decode matrices of erasure patterns that are unions of aligned blocks (e.g. shards {0,1,2,3}) keep the structure.
//     The level L (0 = plain) and the group size of (2) are chosen per matrix by a compile-time op count.
__host__ __device__ constexpr bool bit_subset(int j, int i) { return (j & ~i) == 0; }

template <class MAT, int L>
struct GfXform {
  static constexpr int K = MAT::K, R = MAT::R, B = 1 << L, KB = K / B * B, RB = R / B * B;
  struct Tab {
    uint8_t c[R > 0 ? R : 1][K > 0 ? K : 1];  // transformed matrix, natural (block-major) input order
    uint8_t ord[K > 0 ? K : 1];               // inputs in type-major order (same subset index of every block adjacent)
    signed char top[R > 0 ? R : 1];              // highest plane with a term, -1 = row is zero
  };
  __host__ __device__ static constexpr Tab build() {
    Tab t{};
    for (int r = 0; r < R; r++)
      for (int c = 0; c < K; c++) {
        uint8_t v = 0;
        // C' = Z C Z:  C'[r][c] = XOR over rows i subset-of r and columns j superset-of c (inside their blocks)
        for (int i = (r < RB ? r / B * B : r); i <= r; i++) {
          if (r < RB ? !bit_subset(i % B, r % B) : i != r) continue;
          for (int j = c; j < (c < KB ? c / B * B + B : c + 1); j++) {
            if (c < KB ? !bit_subset(c % B, j % B) : j != c) continue;
            v ^= MAT::coef(i, j);
          }
        }
        t.c[r][c] = v;
      }
    int n = 0;
    for (int pc = L; pc >= 0; pc--)  // subset indices with many bits first: the "block sums" carry the high-degree coefficients
      for (int typ = B - 1; typ >= 0; typ--) {
        int bits = 0;
        for (int q = 0; q < L; q++) bits += (typ >> q) & 1;
        if (bits != pc) continue;
        for (int blk = 0; blk < K / B; blk++) t.ord[n++] = static_cast<uint8_t>(blk * B + typ);
      }
    for (int c = KB; c < K; c++) t.ord[n++] = static_cast<uint8_t>(c);
    for (int r = 0; r < R; r++) {
      int top = -1;
      for (int c = 0; c < K; c++)
        for (int b = 0; b < 8; b++)
          if ((t.c[r][c] >> b) & 1) top = b > top ? b : top;
      t.top[r] = static_cast<signed char>(top);
    }
    return t;
  }
  static constexpr Tab tab = build();

  // index of the XOR combination of group g (inputs ord[GS*g ...]) that feeds row j at Horner plane `plane`
  template <int GS>
  __host__ __device__ static constexpr int combo_index(int j, int g, int plane) {
    int idx = 0;
    for (int q = 0; q < GS; q++)
      if (GS * g + q < K && ((tab.c[j][tab.ord[GS * g + q]] >> plane) & 1)) idx |= 1 << q;
    return idx;
  }
  // ALU-op estimate of run<GS>(): butterflies + distinct multi-input combinations + Horner steps
  template <int GS>
  __host__ __device__ static constexpr int cost() {
    constexpr int G = (K + GS - 1) / GS;
    int ops = (K / B + R / B) * (L * B / 2);
    bool used[G > 0 ? G : 1][1 << GS] = {};
    for (int j = 0; j < R; j++)
      for (int plane = tab.top[j]; plane >= 0; plane--) {
        int n = 0;
        for (int g = 0; g < G; g++) {
          const int idx = combo_index<GS>(j, g, plane);
          if (idx) { n++; used[g][idx] = true; }
        }
        if (plane == tab.top[j]) ops += n > 1 ? n / 2 : 0;
        else ops += 3 + n / 2;  // PRMT + 2 LOP3 absorb one term, every further LOP3 two more
      }
    for (int g = 0; g < G; g++)
      for (int idx = 1; idx < (1 << GS); idx++)
        if (used[g][idx] && (idx & (idx - 1))) ops += (idx == (1 << GS) - 1 && GS == 4) ? 2 : 1;
    return ops;
  }

  template <int GS>
  __host__ __device__ __forceinline__ static void run(const uint32_t (&in)[K], uint32_t (&out)[R]) {
    constexpr int G = (K + GS - 1) / GS, NC = 1 << GS;
    uint32_t y[K];
#pragma unroll
    for (int t = 0; t < K; t++) y[t] = in[t];
    static_for<L>([&](auto l_) {  // subset sums inside every block of B inputs
      constexpr int bit = 1 << decltype(l_)::value;
      static_for<KB>([&](auto t_) {
        constexpr int t = decltype(t_)::value;
        if constexpr ((t % B) & bit) y[t] ^= y[t ^ bit];
      });
    });
    uint32_t cmb[G][NC];
    static_for<G>([&](auto g_) {
      constexpr int g = decltype(g_)::value;
      cmb[g][0] = 0u;
      static_for<NC - 1>([&](auto i_) {
        constexpr int idx = decltype(i_)::value + 1;
        constexpr int low = idx & -idx;  // lowest set bit
        constexpr int q = (low == 1) ? 0 : (low == 2) ? 1 : (low == 4) ? 2 : 3;
        constexpr int pos = GS * g + q;
        if constexpr (pos < K) {
          constexpr int src = tab.ord[pos];
          cmb[g][idx] = cmb[g][idx & (idx - 1)] ^ y[src];  // unused combinations are dead code
        } else {
          cmb[g][idx] = cmb[g][idx & (idx - 1)];
        }
      });
    });
    static_for<R>([&](auto j_) {
      constexpr int j = decltype(j_)::value;
      constexpr int top = tab.top[j];
      uint32_t acc = 0u;
      static_for<(top >= 0 ? top + 1 : 0)>([&](auto s_) {
        constexpr int plane = top - decltype(s_)::value;
        uint32_t terms = 0u;
        static_for<G>([&](auto g_) {
          constexpr int g = decltype(g_)::value;
          constexpr int idx = combo_index<GS>(j, g, plane);
          if constexpr (idx != 0) terms ^= cmb[g][idx];
        });
        if constexpr (plane != top) acc = gf_xtime_add4(acc, terms);
        else acc = terms;
      });
      out[j] = acc;
    });
    static_for<L>([&](auto l_) {  // back from subset sums to the outputs themselves (Z is an involution)
      constexpr int bit = 1 << decltype(l_)::value;
      static_for<RB>([&](auto j_) {
        constexpr int j = decltype(j_)::value;
        if constexpr ((j % B) & bit) out[j] ^= out[j ^ bit];
      });
    });
  }
};

#ifndef MEC_GF_LEVEL
#define MEC_GF_LEVEL -1   // -1: choose the transform level per matrix by op count; 0..3: force it (A/B measurements)
#endif
#ifndef MEC_GF_GROUP
#define MEC_GF_GROUP 0    // 0: choose 3 or 4 inputs per "four Russians" group by op count; 3 / 4: force it
#endif

template <class MAT>  // MAT::K, MAT::R, static constexpr uint8_t MAT::coef(j, t)
struct GfStaticApply {
  static constexpr int K = MAT::K, R = MAT::R;
  template <int L>
  __host__ __device__ static constexpr int level_cost() {
    if constexpr ((1 << L) > K || (1 << L) > R) return 1 << 30;
    else {
      const int c3 = GfXform<MAT, L>::template cost<3>(), c4 = GfXform<MAT, L>::template cost<4>();
      return MEC_GF_GROUP == 3 ? c3 : (MEC_GF_GROUP == 4 ? c4 : (c3 < c4 ? c3 : c4));
    }
  }
  __host__ __device__ static constexpr int choose_level() {
    constexpr int forced = MEC_GF_LEVEL < 0 ? 0 : MEC_GF_LEVEL;
    if (MEC_GF_LEVEL >= 0) return ((1 << forced) > K || (1 << forced) > R) ? 0 : forced;
    int best = 0, bc = level_cost<0>();
    if (level_cost<1>() < bc) { best = 1; bc = level_cost<1>(); }
    if (level_cost<2>() < bc) { best = 2; bc = level_cost<2>(); }
    if (level_cost<3>() < bc) { best = 3; bc = level_cost<3>(); }
    return best;
  }
  static constexpr int kLevel = choose_level();
  using X = GfXform<MAT, kLevel>;
  static constexpr int kGroup = MEC_GF_GROUP == 3 || MEC_GF_GROUP == 4 ? MEC_GF_GROUP
                                                                        : (X::template cost<3>() < X::template cost<4>() ? 3 : 4);
  static constexpr int kOps = kGroup == 3 ? X::template cost<3>() : X::template cost<4>();
  __host__ __device__ __forceinline__ static void run(const uint32_t (&in)[K], uint32_t (&out)[R]) { X::template run<kGroup>(in, out); }
};

// parity rows of reedsolomon.New(K, M): coef(j, t) = M[K + j][t]
template <int K_, int M_>
struct EncodeMatrix {
  static constexpr int K = K_, R = M_;
  static constexpr CodingMatrix<K_, M_> mat = build_coding_matrix<K_, M_>();
  __host__ __device__ static constexpr uint8_t coef(int j, int t) { return mat.v[K_ + j][t]; }
};

// ---------------------------------------------------------------- HighwayHash-256, half state
struct HHHalf {
  uint64_t v0[2], v1[2], m0[2], m1[2];
};

__device__ __forceinline__ uint64_t rot32(uint64_t x) { return (x >> 32) | (x << 32); }
__device__ __forceinline__ uint64_t pack64(uint32_t lo, uint32_t hi) {
  return static_cast<uint64_t>(lo) | (static_cast<uint64_t>(hi) << 32);
}

__device__ __forceinline__ void hh_init(HHHalf& s, const uint64_t (&key)[4], int h) {
  const uint64_t i0a = h ? 0x13198a2e03707344ull : 0xdbe6d5d5fe4cce2full;
  const uint64_t i0b = h ? 0x243f6a8885a308d3ull : 0xa4093822299f31d0ull;
  const uint64_t i1a = h ? 0xbe5466cf34e90c6cull : 0x3bd39e10cb0ef593ull;
  const uint64_t i1b = h ? 0x452821e638d01377ull : 0xc0acf169b5f18a8cull;
  const uint64_t ka = h ? key[2] : key[0], kb = h ? key[3] : key[1];
  s.m0[0] = i0a; s.m0[1] = i0b; s.m1[0] = i1a; s.m1[1] = i1b;
  s.v0[0] = i0a ^ ka; s.v0[1] = i0b ^ kb;
  s.v1[0] = i1a ^ rot32(ka); s.v1[1] = i1b ^ rot32(kb);
}

// ZipperMergeAndAdd(v1 = hi lane, v0 = lo lane): the two 64-bit addends; byte shuffles as PRMTs
__device__ __forceinline__ void hh_zipper(uint64_t hi, uint64_t lo, uint64_t& z1, uint64_t& z0) {
  const uint32_t v0l = static_cast<uint32_t>(lo), v0h = static_cast<uint32_t>(lo >> 32);
  const uint32_t v1l = static_cast<uint32_t>(hi), v1h = static_cast<uint32_t>(hi >> 32);
  // add0 += [v0.b3, v1.b4, v0.b2, v0.b5 | v1.b6, v0.b1, v1.b7, v0.b0]
  // add1 += [v1.b3, v0.b4, v1.b2, v1.b5 | v1.b1, v0.b6, v1.b0, v0.b7]
  // the four bytes both low words take from the high halves are gathered once: 5 PRMTs instead of 6
  const uint32_t x = prmt(v0h, v1h, 0x5041u);  // [v0.b5, v1.b4, v0.b4, v1.b5]
  const uint32_t a0l = prmt(v0l, x, 0x4253u);
  const uint32_t a0h = prmt(v0l, v1h, 0x0716u);
  const uint32_t a1l = prmt(v1l, x, 0x7263u);
  const uint32_t a1h = prmt(v1l, v0h, 0x7061u);
  z0 = pack64(a0l, a0h);
  z1 = pack64(a1l, a1h);
}

// 32 x 32 -> 64 multiply.  MEC_HH_MUL: 0 = mul.wide (IMAD.WIDE), 1 = mul.lo + mul.hi, 2 = mul.wide via PTX with
// an explicit unpack (the plain C form makes ptxas copy the high word through the ALU before the XOR)
#ifndef MEC_HH_MUL
#define MEC_HH_MUL 1
#endif
__device__ __forceinline__ uint64_t hh_mul32(uint32_t a, uint32_t b) {
#if MEC_HH_MUL == 1
  return pack64(a * b, __umulhi(a, b));
#elif MEC_HH_MUL == 2
  uint32_t lo, hi;
  asm("{\n.reg .b64 t;\nmul.wide.u32 t, %2, %3;\nmov.b64 {%0, %1}, t;\n}" : "=r"(lo), "=r"(hi) : "r"(a), "r"(b));
  return pack64(lo, hi);
#else
  return static_cast<uint64_t>(a) * b;
#endif
}

// 64-bit add routed through the FMA pipe: x + y as IMAD.WIDE(y.lo, one, x) + (y.hi << 32).  `one` is
// the value 1 loaded from kernel parameters, so the compiler cannot fold the multiply back into IADD3.
__device__ __forceinline__ uint64_t add64_fma(uint64_t x, uint64_t y, uint32_t one) {
  return static_cast<uint64_t>(static_cast<uint32_t>(y)) * one + x + ((y >> 32) << 32);
}

// HighwayHash Update for the two lanes a thread owns.  MEC_HH_VARIANT moves 64-bit additions from the
// ALU pipe (IADD3/IADD3.X) to the FMA pipe: 0 = none, 1 = the zipper->v1 add, 2 = also v1 += mul0 + packet.
__device__ __forceinline__ void hh_update(HHHalf& s, uint64_t a0, uint64_t a1, uint32_t one = 1u) {
  const uint64_t a[2] = {a0, a1};
  uint64_t m1old[2];
#pragma unroll
  for (int i = 0; i < 2; i++) {
#if MEC_HH_VARIANT >= 2
    s.v1[i] = add64_fma(add64_fma(s.v1[i], a[i], one), s.m0[i], one);
#else
    s.v1[i] += s.m0[i] + a[i];
#endif
    s.m0[i] ^= hh_mul32(static_cast<uint32_t>(s.v1[i]), static_cast<uint32_t>(s.v0[i] >> 32));
    // only the low word of (v0 += mul1) feeds the multiply; the full 64-bit add is merged with the
    // zipper addend below into one 3-input carry chain
    m1old[i] = s.m1[i];
    const uint32_t v0lo = static_cast<uint32_t>(s.v0[i]) + static_cast<uint32_t>(m1old[i]);
    s.m1[i] ^= hh_mul32(v0lo, static_cast<uint32_t>(s.v1[i] >> 32));
  }
  uint64_t z1, z0;
  hh_zipper(s.v1[1], s.v1[0], z1, z0);
  s.v0[0] = s.v0[0] + m1old[0] + z0;
  s.v0[1] = s.v0[1] + m1old[1] + z1;
  hh_zipper(s.v0[1], s.v0[0], z1, z0);
#if MEC_HH_VARIANT >= 1
  s.v1[0] = add64_fma(s.v1[0], z0, one);
  s.v1[1] = add64_fma(s.v1[1], z1, one);
#else
  s.v1[0] += z0;
  s.v1[1] += z1;
#endif
}

// byte `pos` (0..31) of the padded remainder packet for a tail of n (1..31) bytes
template <class GetByte>
__device__ __forceinline__ uint32_t hh_rem_byte(int pos, int n, GetByte&& tail) {
  const int n4 = n & ~3, m4 = n & 3;
  if (pos < n4) return tail(pos);
  if (n & 16) {
    if (pos >= 28) return tail(n - 4 + (pos - 28));
  } else if (m4) {
    if (pos == 16) return tail(n4);
    if (pos == 17) return tail(n4 + (m4 >> 1));
    if (pos == 18) return tail(n4 + m4 - 1);
  }
  return 0u;
}

template <class GetByte>
__device__ __forceinline__ void hh_remainder(HHHalf& s, int h, int n, GetByte&& tail) {
  const uint64_t inc = (static_cast<uint64_t>(n) << 32) + static_cast<uint64_t>(n);
#pragma unroll
  for (int i = 0; i < 2; i++) {
    s.v0[i] += inc;
    const uint32_t lo = static_cast<uint32_t>(s.v1[i]), hi = static_cast<uint32_t>(s.v1[i] >> 32);
    s.v1[i] = pack64(__funnelshift_l(lo, lo, n), __funnelshift_l(hi, hi, n));
  }
  uint64_t a[2] = {0, 0};
  for (int i = 0; i < 16; i++) {
    const uint64_t b = hh_rem_byte(16 * h + i, n, tail);
    a[i >> 3] |= b << (8 * (i & 7));
  }
  hh_update(s, a[0], a[1]);
}

// 10 permute-and-update rounds + modular reduction; thread h==0 returns digest bytes 0..15,
// h==1 bytes 16..31 (as two little-endian u64).  Lanes of a pair must be adjacent (xor 1).
__device__ __forceinline__ void hh_finalize(HHHalf& s, uint64_t& d0, uint64_t& d1) {
#pragma unroll 1
  for (int r = 0; r < 10; r++) {
    const uint64_t p0 = rot32(__shfl_xor_sync(0xffffffffu, s.v0[0], 1));
    const uint64_t p1 = rot32(__shfl_xor_sync(0xffffffffu, s.v0[1], 1));
    hh_update(s, p0, p1);
  }
  const uint64_t a3 = (s.v1[1] + s.m1[1]) & 0x3FFFFFFFFFFFFFFFull;
  const uint64_t a2 = s.v1[0] + s.m1[0];
  const uint64_t a1 = s.v0[1] + s.m0[1];
  const uint64_t a0 = s.v0[0] + s.m0[0];
  d1 = a1 ^ ((a3 << 1) | (a2 >> 63)) ^ ((a3 << 2) | (a2 >> 62));
  d0 = a0 ^ (a2 << 1) ^ (a2 << 2);
}

// ---------------------------------------------------------------- mbarrier + TMA
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  // try_wait suspends the thread for a hardware-bounded time; a transfer that never completes (bad
  // tensor map) traps after ~2^22 retries instead of hanging the GPU.
  uint32_t done = 0;
  for (uint32_t spin = 0; !done; spin++) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.b32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(done)
        : "r"(bar), "r"(parity)
        : "memory");
    if (spin > (1u << 22)) __trap();
  }
}
// one elected lane of a fully converged warp (keeps TMA operands in uniform registers)
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n"
      ".reg .pred P1;\n"
      "elect.sync _|P1, 0xffffffff;\n"
      "selp.b32 %0, 1, 0, P1;\n"
      "}\n"
      : "=r"(pred));
  return pred != 0;
}
__device__ __forceinline__ uint4 lds128(uint32_t addr) {
  uint4 v;
  asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr) : "memory");
  return v;
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
// 2-D tiled TMA load: box lands at `dst` (shared, 128-byte aligned), completion on `bar`
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, int32_t c0, int32_t c1,
                                            uint32_t bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(bar)
      : "memory");
}

// L2 prefetch of a 3-D box (no shared-memory destination, no completion): issued one tile ahead of the load proper so
// that the load finds its lines in L2 instead of waiting out a DRAM round trip under load
__device__ __forceinline__ void tma_prefetch_3d(const CUtensorMap* map, int32_t c0, int32_t c1, int32_t c2) {
  asm volatile("cp.async.bulk.prefetch.tensor.3d.L2.global.tile [%0, {%1, %2, %3}];"
               ::"l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}
__device__ __forceinline__ void tma_prefetch_2d(const CUtensorMap* map, int32_t c0, int32_t c1) {
  asm volatile("cp.async.bulk.prefetch.tensor.2d.L2.global.tile [%0, {%1, %2}];"
               ::"l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1)
               : "memory");
}
// consumer release: one arrival on a plain (no transaction bytes) mbarrier
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}

// 3-D tiled TMA load (x, block, shard row)
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* map, int32_t c0, int32_t c1, int32_t c2,
                                            uint32_t bar) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(c2), "r"(bar)
      : "memory");
}

}  // namespace mec
