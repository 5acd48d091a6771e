// crc.cuh — object checksums of the PutObject stream (internal/hash/checksum.go:64-73, internal/hash/crc.go): CRC32 (IEEE),
// CRC32C (Castagnoli) and CRC64NVME, the three mergeable types (ChecksumType.CanMerge, checksum.go:277).  hash.Reader computes
// them over the same bytes Erasure.Encode reads (cmd/object-handlers.go:1964-2083); here they are computed on the copy of the
// object that is already in HBM for the encode.
//
// A CRC is sequential per byte but linear over GF(2): crc(A || B) = crc(A) * x^(8|B|) mod P  xor  crc(B) — exactly the merge
// MinIO's own Checksum.AddPart performs for multipart objects (crc32Combine / crc64Combine, crc.go:98-220).  So: every thread
// runs the byte-wise table CRC over its own 1 KiB chunk (tables in shared memory), the 256 partials of a CTA are merged by a
// tree of multiplications modulo P (lengths are powers of two, the factors x^(8*2^i) mod P are constants), one partial per
// 256 KiB region goes to global memory and a single CTA folds those.  All three CRCs are reflected, init and xorout all-ones;
// the 32-bit ones are carried in the low half of 64-bit words and use the same code as the 64-bit one.
#pragma once
#include <cstdint>

namespace mec {

constexpr int kCrcTypes = 3;                 // index 0 = CRC32 (IEEE), 1 = CRC32C, 2 = CRC64NVME
constexpr int kCrcChunk = 1024;              // bytes per thread
constexpr int kCrcThreads = 256;             // threads per CTA -> 256 KiB per CTA pass
constexpr int64_t kCrcRegion = static_cast<int64_t>(kCrcChunk) * kCrcThreads;

struct CrcSpec {
  uint64_t poly;  // reflected polynomial
  int bits;       // 32 or 64
};
__host__ __device__ constexpr CrcSpec crc_spec(int t) {
  return t == 0 ? CrcSpec{0xEDB88320ull, 32} : (t == 1 ? CrcSpec{0x82F63B78ull, 32} : CrcSpec{0x9A6C9329AC4BC9B5ull, 64});
}
__host__ __device__ constexpr uint64_t crc_mask(int bits) { return bits == 64 ? ~0ull : ((1ull << bits) - 1); }

// a(x) * b(x) mod P in the reflected representation (bit `bits-1` is x^0): the shift-and-add product zlib's multmodp uses
__host__ __device__ inline uint64_t crc_mulmod(uint64_t a, uint64_t b, uint64_t poly, int bits) {
  uint64_t m = 1ull << (bits - 1), p = 0;
  for (int i = 0; i < bits; i++) {
    if (a & m) p ^= b;
    m >>= 1;
    b = (b & 1) ? (b >> 1) ^ poly : b >> 1;
  }
  return p;
}

struct CrcTables {
  uint64_t byte_tab[kCrcTypes][256];  // classic byte-at-a-time table
  uint64_t xp8[kCrcTypes][64];        // x^(8 * 2^i) mod P
};

inline void crc_build_tables(CrcTables* t) {
  for (int ty = 0; ty < kCrcTypes; ty++) {
    const CrcSpec sp = crc_spec(ty);
    for (int v = 0; v < 256; v++) {
      uint64_t c = static_cast<uint64_t>(v);
      for (int k = 0; k < 8; k++) c = (c & 1) ? (c >> 1) ^ sp.poly : c >> 1;
      t->byte_tab[ty][v] = c;
    }
    uint64_t p = 1ull << (sp.bits - 9);  // x^8: bit `bits-1` is x^0 in the reflected form
    for (int i = 0; i < 64; i++) {
      t->xp8[ty][i] = p;
      p = crc_mulmod(p, p, sp.poly, sp.bits);
    }
  }
}

// x^(8n) mod P
__host__ __device__ inline uint64_t crc_xpow8(const uint64_t* xp8, int64_t n, uint64_t poly, int bits) {
  uint64_t r = 1ull << (bits - 1);  // x^0
  for (int i = 0; n > 0 && i < 64; i++, n >>= 1)
    if (n & 1) r = crc_mulmod(r, xp8[i], poly, bits);
  return r;
}
// Checksum.AddPart: crc of A || B from crc(A), crc(B), |B|
__host__ __device__ inline uint64_t crc_combine(const uint64_t* xp8, uint64_t c1, uint64_t c2, int64_t len2, uint64_t poly, int bits) {
  if (len2 <= 0) return c1;
  return crc_mulmod(crc_xpow8(xp8, len2, poly, bits), c1, poly, bits) ^ c2;
}

struct CrcParams {
  const uint8_t* src;
  int64_t len;
  int which;                 // bit t set = compute type t
  const CrcTables* tables;   // device copy
  uint64_t* partial;         // [nregions][kCrcTypes]
  int64_t nregions;
  uint64_t* out;             // [kCrcTypes]
};

// Object checksums of the PUTs of a merged coalescer batch (mec_batcher_encode_crc).  A request's bytes are two segments of the
// staged buffer (its full blocks, then its short last block elsewhere), each cut into regions of at most kCrcRegion bytes that
// never cross a segment edge: one work item per region, the items of a request consecutive and in stream order.
struct CrcWork {
  int64_t off;    // first byte of the region, from CrcSegParams::base (any alignment)
  int32_t len;    // 1 .. kCrcRegion; kCrcRegion for every region of a segment but its last
  int32_t which;  // types its request asked for
};
struct CrcReq {
  int32_t w0, w1;  // the request's work items [w0, w1)
  int32_t which;   // 0: no checksums for this request (no items)
  int32_t pad;
};
struct CrcSegParams {
  const uint8_t* base;
  const CrcWork* work;
  const CrcReq* reqs;
  int64_t nwork;
  int nreq;
  int which;                 // union of the requests' masks: the byte tables to load
  const CrcTables* tables;   // device copy
  uint64_t* partial;         // [nwork][kCrcTypes]
  uint64_t* out;             // [nreq][kCrcTypes], 0 where the request did not ask
};
constexpr int kCrcFoldThreads = 128;  // four requests per CTA of the fold kernel, one warp each
static_assert(kCrcRegion == (1 << 18), "xp8[ty][18] is the factor of a whole region");

#ifdef __CUDACC__
// CRCs (types in `which`) of the region src[0, rlen), rlen <= kCrcRegion, by all kCrcThreads threads of the CTA: per-thread chunk
// CRCs, then a tree merge in shared memory; thread 0 writes part[ty].  Every thread of the CTA must call it with the same arguments.
__device__ inline void crc_region(const uint8_t* src, int64_t rlen, int which, const uint64_t (*s_tab)[256], uint64_t* s_part,
                                  const CrcTables* tables, uint64_t* part) {
  const int tid = threadIdx.x;
  int64_t n = rlen - static_cast<int64_t>(tid) * kCrcChunk;
  n = n < 0 ? 0 : (n > kCrcChunk ? kCrcChunk : n);
  uint64_t crc[kCrcTypes];
#pragma unroll
  for (int ty = 0; ty < kCrcTypes; ty++) crc[ty] = crc_mask(crc_spec(ty).bits);  // init: all ones
  const uint8_t* q = src + static_cast<int64_t>(tid) * kCrcChunk;
  auto step = [&](uint32_t b) {
#pragma unroll
    for (int ty = 0; ty < kCrcTypes; ty++)
      if (which & (1 << ty)) crc[ty] = s_tab[ty][(crc[ty] ^ b) & 0xffu] ^ (crc[ty] >> 8);
  };
  // bytes up to the first 16-byte boundary one at a time, then 16-byte loads (a chunk of a misaligned segment is misaligned too)
  const int64_t head = (16 - static_cast<int64_t>(reinterpret_cast<uintptr_t>(q) & 15)) & 15;
  int64_t i = 0;
  for (; i < n && i < head; i++) step(q[i]);
  for (; i + 16 <= n; i += 16) {
    const uint4 v = __ldg(reinterpret_cast<const uint4*>(q + i));
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int k = 0; k < 16; k++) step((w[k >> 2] >> (8 * (k & 3))) & 0xffu);
  }
  for (; i < n; i++) step(q[i]);
  // tree merge: at level `lv` thread t (t % 2^(lv+1) == 0) absorbs thread t + 2^lv; lengths follow from the region length
#pragma unroll
  for (int ty = 0; ty < kCrcTypes; ty++) {
    if (!(which & (1 << ty))) continue;
    const CrcSpec sp = crc_spec(ty);
    uint64_t mine = crc[ty] ^ crc_mask(sp.bits);  // xorout
    __syncthreads();
    for (int lv = 0; (1 << lv) < kCrcThreads; lv++) {
      s_part[tid] = mine;
      __syncthreads();
      const int span = 1 << lv;
      if ((tid & (2 * span - 1)) == 0) {
        // bytes covered by the right-hand subtree [tid + span, tid + 2 span) inside this region
        int64_t rb = rlen - static_cast<int64_t>(tid + span) * kCrcChunk;
        rb = rb < 0 ? 0 : (rb > static_cast<int64_t>(span) * kCrcChunk ? static_cast<int64_t>(span) * kCrcChunk : rb);
        if (rb > 0) mine = crc_combine(tables->xp8[ty], mine, s_part[tid + span], rb, sp.poly, sp.bits);
      }
      __syncthreads();
    }
    if (tid == 0) part[ty] = mine;
  }
}

// one CTA pass = one 256 KiB region of p.src
__global__ void __launch_bounds__(kCrcThreads) crc_regions_kernel(const CrcParams p) {
  __shared__ uint64_t s_tab[kCrcTypes][256];
  __shared__ uint64_t s_part[kCrcThreads];
  const int tid = threadIdx.x;
  for (int ty = 0; ty < kCrcTypes; ty++)
    if (p.which & (1 << ty)) s_tab[ty][tid] = p.tables->byte_tab[ty][tid];
  __syncthreads();
  for (int64_t rg = blockIdx.x; rg < p.nregions; rg += gridDim.x) {
    const int64_t rlen = (p.len - rg * kCrcRegion) > kCrcRegion ? kCrcRegion : (p.len - rg * kCrcRegion);
    crc_region(p.src + rg * kCrcRegion, rlen, p.which, s_tab, s_part, p.tables, p.partial + rg * kCrcTypes);
  }
}

// one CTA pass = one work item of a merged batch
__global__ void __launch_bounds__(kCrcThreads) crc_seg_regions_kernel(const CrcSegParams p) {
  __shared__ uint64_t s_tab[kCrcTypes][256];
  __shared__ uint64_t s_part[kCrcThreads];
  const int tid = threadIdx.x;
  for (int ty = 0; ty < kCrcTypes; ty++)
    if (p.which & (1 << ty)) s_tab[ty][tid] = p.tables->byte_tab[ty][tid];
  __syncthreads();
  for (int64_t w = blockIdx.x; w < p.nwork; w += gridDim.x) {
    const CrcWork wk = p.work[w];
    crc_region(p.base + wk.off, wk.len, wk.which, s_tab, s_part, p.tables, p.partial + w * kCrcTypes);
  }
}

// one warp per request: each lane folds a contiguous run of the request's items in order (a whole region appended = one product with
// the constant x^(8 * kCrcRegion)), then the 32 runs are merged by a shuffle tree
__global__ void __launch_bounds__(kCrcFoldThreads) crc_seg_fold_kernel(const CrcSegParams p) {
  const int q = (blockIdx.x * kCrcFoldThreads + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (q >= p.nreq) return;  // whole warps
  const CrcReq rq = p.reqs[q];
  const int nw = rq.w1 - rq.w0, per = (nw + 31) / 32;
  const int a = rq.w0 + min(nw, lane * per), e = rq.w0 + min(nw, (lane + 1) * per);
  for (int ty = 0; ty < kCrcTypes; ty++) {
    if (!(rq.which & (1 << ty))) {
      if (lane == 0) p.out[q * kCrcTypes + ty] = 0;
      continue;
    }
    const CrcSpec sp = crc_spec(ty);
    const uint64_t* xp8 = p.tables->xp8[ty];
    uint64_t acc = 0;
    int64_t alen = 0;
    for (int w = a; w < e; w++) {
      const int64_t len = p.work[w].len;
      const uint64_t c = p.partial[static_cast<int64_t>(w) * kCrcTypes + ty];
      acc = alen == 0 ? c : crc_mulmod(len == kCrcRegion ? xp8[18] : crc_xpow8(xp8, len, sp.poly, sp.bits), acc, sp.poly, sp.bits) ^ c;
      alen += len;
    }
    for (int span = 1; span < 32; span <<= 1) {
      const uint64_t rc = __shfl_down_sync(0xffffffffu, acc, span);
      const int64_t rl = __shfl_down_sync(0xffffffffu, alen, span);
      if ((lane & (2 * span - 1)) == 0 && rl > 0) {
        acc = alen == 0 ? rc : crc_combine(xp8, acc, rc, rl, sp.poly, sp.bits);
        alen += rl;
      }
    }
    if (lane == 0) p.out[q * kCrcTypes + ty] = acc;
  }
}

// fold the region partials (region r covers min(kCrcRegion, len - r * kCrcRegion) bytes): tree over 256 threads, then serial
__global__ void __launch_bounds__(kCrcThreads) crc_fold_kernel(const CrcParams p) {
  __shared__ uint64_t s_part[kCrcThreads];
  __shared__ int64_t s_len[kCrcThreads];
  const int tid = threadIdx.x;
  for (int ty = 0; ty < kCrcTypes; ty++) {
    if (!(p.which & (1 << ty))) { if (tid == 0) p.out[ty] = 0; continue; }
    const CrcSpec sp = crc_spec(ty);
    // each thread folds a contiguous run of regions serially, then the runs are merged in order
    const int64_t per = (p.nregions + kCrcThreads - 1) / kCrcThreads;
    const int64_t r0 = static_cast<int64_t>(tid) * per, r1 = (r0 + per < p.nregions) ? r0 + per : p.nregions;
    uint64_t acc = 0;
    int64_t alen = 0;
    for (int64_t r = r0; r < r1; r++) {
      const int64_t rl = (p.len - r * kCrcRegion) > kCrcRegion ? kCrcRegion : (p.len - r * kCrcRegion);
      acc = alen == 0 ? p.partial[r * kCrcTypes + ty] : crc_combine(p.tables->xp8[ty], acc, p.partial[r * kCrcTypes + ty], rl, sp.poly, sp.bits);
      alen += rl;
    }
    s_part[tid] = acc;
    s_len[tid] = alen;
    __syncthreads();
    if (tid == 0) {
      uint64_t tot = 0;
      int64_t tl = 0;
      for (int t = 0; t < kCrcThreads; t++) {
        if (s_len[t] == 0) continue;
        tot = tl == 0 ? s_part[t] : crc_combine(p.tables->xp8[ty], tot, s_part[t], s_len[t], sp.poly, sp.bits);
        tl += s_len[t];
      }
      p.out[ty] = tot;
    }
    __syncthreads();
  }
}
#endif

}  // namespace mec
