// ec_small.cuh — the latency form of the fused Reed-Solomon + HighwayHash-256 kernel (sm_90a).
//
// The throughput kernel (ec_kernel.cuh) gives every erasure block to ONE warp: its lanes multiply a 256-byte tile, then the same
// lanes hash it, 341 times per 1 MiB block — ~0.45 ms however few blocks the launch brings (a PutObject of one small object, the
// 1 MiB-per-iteration loop of cmd/erasure-encode.go:76-108, a merged batch of a few dozen requests), with most SMs idle.
// HighwayHash is a serial chain per shard, so a block cannot be finished faster than 2731 dependent packet updates; what CAN be
// removed is everything else on that critical path.  Here a CTA owns one block and is warp-specialised:
//   * GF warps (three or four, one 8-byte column per thread of a 768- or 1024-byte super-tile): fetch with cp.async (16-byte chunks
//     from the 16-byte boundary below each row, zero-filled beyond the row's valid bytes = Split's padding), three stages deep;
//     re-align, store the aligned rows, multiply, store the output rows (shared + global);
//   * hash warps (two lanes per shard stream, 16 streams per warp): wait for a super-tile, run its 24 or 32 packet updates back
//     to back, hand the buffer back.  Nothing but the hash chain is on their path.
// full/empty mbarriers pair the two roles over two aligned buffers.  Same arithmetic, same digests, same outputs as the
// throughput kernel — the engine picks this one when a launch has fewer blocks than would fill the GPU (ec_engine.cu).
#pragma once
#include "ec_kernel.cuh"

namespace mec {

// GW = GF warps per CTA: three beside one hash warp (up to 16 streams; 55 KB of shared memory for RS(12,4): four CTAs per SM),
// four beside two or three (wider stripes have more GF and fetch work per column than two GF warps keep up with).  A pipeline stage ("super-tile") is 256 bytes of every shard per GF warp.
__host__ __device__ constexpr int small_super(int gw) { return 256 * gw; }
__host__ __device__ constexpr int small_chunks(int gw) { return small_super(gw) / 16 + 1; }  // 16-byte chunks per row and stage (lead <= 15 bytes + funnel slack)
__host__ __device__ constexpr int small_raw_pitch(int gw) { return small_chunks(gw) * 16 + 16; }
__host__ __device__ constexpr int small_row_pitch(int gw) { return small_super(gw) + 32; }  // = 32 mod 128: a quarter-warp's four streams on disjoint banks
constexpr int kSmallStages = 3;
__host__ __device__ constexpr int small_gf_warps(int nstreams) { return (2 * nstreams + 31) / 32 == 1 ? 3 : 4; }

struct SmallRow {
  const uint8_t* base16;  // 16-byte boundary at or below the row's first byte
  int32_t lead;           // bytes between base16 and the first byte
  int32_t valid;          // bytes of the row that exist (the rest of S reads as zero)
};

__host__ __device__ constexpr int small_hash_warps(int nstreams) { return (2 * nstreams + 31) / 32; }
__host__ __device__ constexpr uint32_t small_smem_bytes(int k, int r, bool dynamic_gf, int gw) {
  uint32_t b = static_cast<uint32_t>(kSmallStages * k) * small_raw_pitch(gw) + static_cast<uint32_t>(2 * (k + r)) * small_row_pitch(gw);
  b += 64 + static_cast<uint32_t>(kMaxK) * sizeof(SmallRow);
  if (dynamic_gf) b += static_cast<uint32_t>(k) * ((r + kRChunk - 1) / kRChunk) * kRChunk * 8 * 4;
  return b;
}

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, int32_t src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
template <int N>
__device__ __forceinline__ void gf_warps_sync() { asm volatile("bar.sync 1, %0;" ::"n"(N) : "memory"); }

template <class GF, int GW>
__global__ void __launch_bounds__(256, 2) small_rs_hh_kernel(const __grid_constant__ FusedParams p) {
  constexpr int kSmallSuper = small_super(GW), kSmallChunks = small_chunks(GW), kSmallRawPitch = small_raw_pitch(GW),
                kSmallRowPitch = small_row_pitch(GW), kSmallGfThreads = 32 * GW;
  extern __shared__ __align__(128) uint8_t smem[];
  const int k = GF::kIsStatic ? GF::K : p.k;
  const int r = GF::kIsStatic ? GF::R : p.r;
  const int nstreams = k + r;
  const int tid = threadIdx.x;
  const int nht = static_cast<int>(blockDim.x) - kSmallGfThreads;  // hash threads (whole warps), then the GF threads
  uint8_t* s_raw = smem;                                                                   // [stage][k][raw pitch]
  uint8_t* s_rows = s_raw + static_cast<uint32_t>(kSmallStages * k) * kSmallRawPitch;       // [2][k + r][row pitch]: inputs, then outputs
  uint64_t* bars = reinterpret_cast<uint64_t*>(s_rows + static_cast<uint32_t>(2 * nstreams) * kSmallRowPitch);  // full[2], empty[2]
  SmallRow* rows = reinterpret_cast<SmallRow*>(bars + 8);
  uint32_t* s_masks = reinterpret_cast<uint32_t*>(rows + kMaxK);
  const int rpad = (r + kRChunk - 1) / kRChunk * kRChunk;

  const int64_t b = blockIdx.x;
  // per-block geometry: the short last frames of many part files, or the blocks of many PutObjects, ride in one launch
  const bool is_tail = p.tail_block == b;
  const int32_t S = p.blocks != nullptr ? p.blocks[b].S : (p.block_len != nullptr ? p.block_len[b] : (is_tail ? p.tail_S : p.S));
  const int nst = (S + kSmallSuper - 1) / kSmallSuper;
  // a launch of mixed erasure patterns: this block's own decode plan.  The launch's r (the largest of its plans) sizes shared
  // memory, the digest and output layouts; only rows j < br are computed, stored and hashed here
  int br = r;
  const SmallPattern* pat = nullptr;
  if constexpr (!GF::kIsStatic) {
    if (p.block_pattern != nullptr) {
      pat = p.patterns + p.block_pattern[b];
      br = pat->r;
    }
  }

  if (tid == 0) {
    mbar_init(smem_u32(&bars[0]), kSmallGfThreads);
    mbar_init(smem_u32(&bars[1]), kSmallGfThreads);
    mbar_init(smem_u32(&bars[2]), static_cast<uint32_t>(nht));
    mbar_init(smem_u32(&bars[3]), static_cast<uint32_t>(nht));
    fence_barrier_init();
  }
  if (tid < k) {
    const uint8_t* a = p.in_ptr[tid] + b * p.in_block_stride;
    int64_t valid = p.in_limit - static_cast<int64_t>(tid) * p.in_shard_step;
    if (p.blocks != nullptr) {
      a = p.in_ptr[0] + p.blocks[b].in_off + static_cast<int64_t>(tid) * S;
      valid = static_cast<int64_t>(p.blocks[b].bytes) - static_cast<int64_t>(tid) * S;
    } else if (is_tail && p.tail_in_off >= 0) {
      a = p.in_ptr[0] + p.tail_in_off + static_cast<int64_t>(tid) * S;
      valid = static_cast<int64_t>(p.tail_bytes) - static_cast<int64_t>(tid) * S;
    }
    valid = valid < 0 ? 0 : (valid > S ? S : valid);
    SmallRow rw;
    rw.base16 = reinterpret_cast<const uint8_t*>(reinterpret_cast<uintptr_t>(a) & ~static_cast<uintptr_t>(15));
    rw.lead = static_cast<int32_t>(reinterpret_cast<uintptr_t>(a) & 15);
    rw.valid = static_cast<int32_t>(valid);
    rows[tid] = rw;
  }
  if constexpr (!GF::kIsStatic) {
    for (int i = tid; i < k * rpad * 8; i += blockDim.x) {
      const int bit = i & 7, j = (i >> 3) % rpad, t = (i >> 3) / rpad;
      const uint32_t c = j < br ? (pat != nullptr ? pat->coef[j][t] : p.coef[j][t]) : 0u;
      s_masks[i] = 0u - ((c >> bit) & 1u);
    }
  }
  __syncthreads();

  if (tid >= nht) {
    // ------------------------------------------------------------------ GF warps
    const int gt = tid - nht;
    auto issue = [&](int i) {
      if (i < nst) {
        uint8_t* dst = s_raw + static_cast<uint32_t>((i % kSmallStages) * k) * kSmallRawPitch;
        for (int c = gt; c < k * kSmallChunks; c += kSmallGfThreads) {
          const int t = c / kSmallChunks, q = c - t * kSmallChunks;
          const SmallRow rw = rows[t];
          const int64_t off = static_cast<int64_t>(i) * kSmallSuper + 16 * q;  // from base16; the row's bytes are [lead, lead + valid)
          int64_t n = static_cast<int64_t>(rw.lead) + rw.valid - off;
          n = n < 0 ? 0 : (n > 16 ? 16 : n);
          cp_async16(smem_u32(dst + static_cast<uint32_t>(t) * kSmallRawPitch + 16 * q), rw.base16 + (n > 0 ? off : 0), static_cast<int32_t>(n));
        }
      }
      cp_async_commit();  // always: keeps the group count in step with the stage count
    };
    issue(0);
    issue(1);
#pragma unroll 1
    for (int i = 0; i < nst; i++) {
      cp_async_wait<1>();  // this thread's chunks of stage i have landed
      gf_warps_sync<kSmallGfThreads>();     // ... and everybody else's; every GF thread is also done with stage i - 1, whose raw buffer is refilled next
      issue(i + 2);
      const int buf = i & 1;
      if (i >= 2) mbar_wait(smem_u32(&bars[2 + buf]), static_cast<uint32_t>(((i >> 1) - 1) & 1));  // hash warps are done with tile i - 2
      const uint8_t* rcol = s_raw + static_cast<uint32_t>((i % kSmallStages) * k) * kSmallRawPitch + gt * 8;
      uint8_t* ccol = s_rows + static_cast<uint32_t>(buf * nstreams) * kSmallRowPitch + gt * 8;
      const int64_t xg = static_cast<int64_t>(i) * kSmallSuper + gt * 8;
      uint8_t* gout = p.out + b * r * p.out_pitch + xg;
      const bool full = xg + 8 <= S, part = xg < S && !full;
      auto store_out = [&](int j, uint2 o) {
        *reinterpret_cast<uint2*>(ccol + static_cast<uint32_t>(k + j) * kSmallRowPitch) = o;
        uint8_t* gp = gout + j * p.out_pitch;
        if (full) {
          *reinterpret_cast<uint2*>(gp) = o;
        } else if (part) {
          const uint64_t w = pack64(o.x, o.y);
          for (int q = 0; q < 8 && xg + q < S; q++) gp[q] = static_cast<uint8_t>(w >> (8 * q));
        }
      };
      if constexpr (GF::kIsStatic) {
        constexpr int K = GF::K, R = GF::R;
        uint32_t lo[K], hi[K];
        static_for<K>([&](auto t_) {
          constexpr int t = decltype(t_)::value;
          const uint2 v = load_col_rt(rcol + t * kSmallRawPitch, static_cast<uint32_t>(rows[t].lead));
          lo[t] = v.x; hi[t] = v.y;
          *reinterpret_cast<uint2*>(ccol + t * kSmallRowPitch) = v;
        });
        if constexpr (R > 0) {
          uint32_t olo[R], ohi[R];
          GfStaticApply<typename GF::Mat>::run(lo, olo);
          GfStaticApply<typename GF::Mat>::run(hi, ohi);
#pragma unroll
          for (int j = 0; j < R; j++) store_out(j, make_uint2(olo[j], ohi[j]));
        }
      } else {
        constexpr int RC = GF::RC;
        for (int j0 = 0; j0 < (br > 0 ? br : 1); j0 += RC) {
          uint32_t pl[RC][8], ph[RC][8];
#pragma unroll
          for (int j = 0; j < RC; j++)
#pragma unroll
            for (int q = 0; q < 8; q++) { pl[j][q] = 0u; ph[j][q] = 0u; }
#pragma unroll 2
          for (int t = 0; t < k; t++) {
            const uint2 v = load_col_rt(rcol + t * kSmallRawPitch, static_cast<uint32_t>(rows[t].lead));
            if (j0 == 0) *reinterpret_cast<uint2*>(ccol + t * kSmallRowPitch) = v;
            if (br == 0) continue;
            const uint4* mk = reinterpret_cast<const uint4*>(s_masks + (t * rpad + j0) * 8);
#pragma unroll
            for (int j = 0; j < RC; j++) {
              const uint4 m0 = mk[2 * j], m1 = mk[2 * j + 1];
              pl[j][0] ^= v.x & m0.x; ph[j][0] ^= v.y & m0.x;
              pl[j][1] ^= v.x & m0.y; ph[j][1] ^= v.y & m0.y;
              pl[j][2] ^= v.x & m0.z; ph[j][2] ^= v.y & m0.z;
              pl[j][3] ^= v.x & m0.w; ph[j][3] ^= v.y & m0.w;
              pl[j][4] ^= v.x & m1.x; ph[j][4] ^= v.y & m1.x;
              pl[j][5] ^= v.x & m1.y; ph[j][5] ^= v.y & m1.y;
              pl[j][6] ^= v.x & m1.z; ph[j][6] ^= v.y & m1.z;
              pl[j][7] ^= v.x & m1.w; ph[j][7] ^= v.y & m1.w;
            }
          }
#pragma unroll
          for (int j = 0; j < RC; j++) {
            if (j0 + j >= br) break;
            uint32_t al = pl[j][7], ah = ph[j][7];
#pragma unroll
            for (int q = 6; q >= 0; q--) {
              al = gf_xtime_add4(al, pl[j][q]);
              ah = gf_xtime_add4(ah, ph[j][q]);
            }
            store_out(j0 + j, make_uint2(al, ah));
          }
        }
      }
      mbar_arrive(smem_u32(&bars[buf]));  // tile i is in the aligned buffer (release: the stores above are visible to the waiters)
    }
    cp_async_wait<0>();
    return;
  }

  // -------------------------------------------------------------------- hash warps: two lanes per stream
  const int s = tid >> 1, h = tid & 1;
  int nhash = GF::kHashOut == 1 ? nstreams : (GF::kHashOut == 0 ? k : p.nhash);
  if constexpr (!GF::kIsStatic)
    if (pat != nullptr && nhash > k) nhash = k + br;
  const bool live = p.digests != nullptr && s < nhash;
  const bool is_out = s >= k;
  HHHalf hs;
  hh_init(hs, p.key, h);
  const int npk = S >> 5, rem = S & 31;
#pragma unroll 1
  for (int i = 0; i < nst; i++) {
    const int buf = i & 1;
    mbar_wait(smem_u32(&bars[buf]), static_cast<uint32_t>((i >> 1) & 1));
    if (live) {
      const uint8_t* row = s_rows + static_cast<uint32_t>(buf * nstreams + s) * kSmallRowPitch;
      const uint32_t addr = smem_u32(row) + 16u * h;
      const int cnt = npk - i * (kSmallSuper / 32);
      if (cnt >= kSmallSuper / 32) {
#pragma unroll 8
        for (int q = 0; q < kSmallSuper / 32; q++) {
          const uint4 v = lds128(addr + 32 * q);
          hh_update(hs, pack64(v.x, v.y), pack64(v.z, v.w));
        }
      } else {
#pragma unroll 1
        for (int q = 0; q < cnt; q++) {
          const uint4 v = lds128(addr + 32 * q);
          hh_update(hs, pack64(v.x, v.y), pack64(v.z, v.w));
        }
      }
      if (i == nst - 1 && rem) {
        const uint8_t* tail = row + (npk * 32 - i * kSmallSuper);
        hh_remainder(hs, h, rem, [&](int idx) -> uint32_t { return tail[idx]; });
      }
    }
    mbar_arrive(smem_u32(&bars[2 + buf]));
  }
  uint64_t d0, d1;
  hh_finalize(hs, d0, d1);  // all lanes of the warp take part in the shuffles
  if (live) {
    uint64_t* dg = reinterpret_cast<uint64_t*>(p.digests + (b * nstreams + s) * 32 + 16 * h);
    dg[0] = d0;
    dg[1] = d1;
    if (!is_out && p.corrupt != nullptr && p.expect_ptr[s] != nullptr) {
      const uint8_t* ex = p.expect_ptr[s] + b * p.expect_block_stride + 16 * h;
      uint64_t e0 = 0, e1 = 0;
      for (int q = 0; q < 8; q++) {
        e0 |= static_cast<uint64_t>(ex[q]) << (8 * q);
        e1 |= static_cast<uint64_t>(ex[8 + q]) << (8 * q);
      }
      if (e0 != d0 || e1 != d1) p.corrupt[b * k + s] = 1;
    }
  }
}

}  // namespace mec
