// batch_copy.cuh — gather / scatter kernels of the cross-request coalescer (mec_batcher).
// A merged batch of hundreds of small PutObject calls cannot afford a handful of cudaMemcpy* calls per request: at ~4 us of
// driver time each, the worker thread tops out near 25 k requests/s.  Page-locked host memory is mapped into the device's
// address space (UVA), so two kernels move everything instead, driven by one descriptor table per batch:
//   gather : object bytes of every request, host -> the merged staging buffer (full blocks contiguous, tails behind them)
//   scatter: digest + shard of every (request, drive, block) straight into the caller's part-file images — the frame
//            assembly of streamingBitrotWriter.Write (cmd/bitrot-streaming.go:57-69), Split's zero padding included —
//            or, for the scatter-gather form, the data-shard digests into the caller's digest array.
// Host frames start at arbitrary byte offsets (a frame is 32 + S bytes); stores are issued 16-byte aligned on the DESTINATION
// (whole 128-byte PCIe writes per warp) and the source is re-aligned in registers.
#pragma once
#include <cstdint>
#include "whole_hash.cuh"  // WholeStream

namespace mec {

constexpr int kBatchMaxFiles = 32;   // drives per erasure set the batcher accepts (MinIO sets have <= 16)

struct BatchReqDesc {
  const uint8_t* src;                // host (mapped): the caller's object bytes
  int64_t len;
  uint8_t* files[kBatchMaxFiles];    // host (mapped): part-file images, nullptr = offline / not wanted
  uint8_t* data_digests;             // host (mapped) or nullptr: [block][k][32]
  int64_t full0;                     // merged layout: slot of the request's first full block
  int64_t tail_slot;                 // slot of its tail block (parity rows / digests), -1 = none
  int64_t tail_src_off;              // byte offset of the tail block in the staging buffer
  int32_t with_data;                 // 1: data drives get complete frames too
  int32_t pad;
};

struct BatchCopyParams {
  const BatchReqDesc* reqs;          // host (mapped) table
  int nreq, k, m;
  int64_t bs, S, pitch;
  uint8_t* staged;                   // device: merged object bytes
  const uint8_t* parity;             // device: parity rows, slot s row j at (s*m + j)*pitch
  const uint8_t* digests;            // device: [slot][k+m][32]
};

// 16 bytes from an arbitrarily aligned source (4-byte aligned loads + funnel shifts)
__device__ __forceinline__ uint4 load16_any(const uint8_t* p) {
  const uintptr_t a = reinterpret_cast<uintptr_t>(p);
  if ((a & 15) == 0) return *reinterpret_cast<const uint4*>(p);
  const uint32_t* w = reinterpret_cast<const uint32_t*>(a & ~static_cast<uintptr_t>(3));
  const uint32_t sh = static_cast<uint32_t>(a & 3) * 8;
  const uint32_t w0 = w[0], w1 = w[1], w2 = w[2], w3 = w[3];
  if (sh == 0) return make_uint4(w0, w1, w2, w3);
  const uint32_t w4 = w[4];
  return make_uint4(__funnelshift_r(w0, w1, sh), __funnelshift_r(w1, w2, sh), __funnelshift_r(w2, w3, sh), __funnelshift_r(w3, w4, sh));
}

// copy n bytes; dst may be misaligned: byte head up to the first 16-byte boundary of dst, 16-byte body, byte tail.
// The source must be readable up to 4 bytes past its end rounded up to a word (device staging buffers are padded; host
// sources are read exactly, see `exact_src`).
__device__ __forceinline__ void cta_copy(uint8_t* dst, const uint8_t* src, int64_t n, bool exact_src) {
  const int tid = threadIdx.x, nt = blockDim.x;
  const int64_t head = n < 16 ? n : ((16 - (reinterpret_cast<uintptr_t>(dst) & 15)) & 15);
  for (int64_t i = tid; i < head; i += nt) dst[i] = src[i];
  int64_t body = (n - head) / 16;
  if (exact_src && body > 0 && (reinterpret_cast<uintptr_t>(src + head) & 3) != 0) body--;  // the last funnel would read 1-3 bytes past the source
  for (int64_t q = tid; q < body; q += nt) *reinterpret_cast<uint4*>(dst + head + q * 16) = load16_any(src + head + q * 16);
  for (int64_t i = head + body * 16 + tid; i < n; i += nt) dst[i] = src[i];
}
// Host -> device copy for sources in mapped host memory.  SM loads over PCIe are worth their latency only as whole 128-byte
// requests, and host frames start at arbitrary (even) offsets: the source is therefore read in 16-byte vectors aligned on the
// SOURCE (every warp load = 512 contiguous bytes) into a shared-memory stage, and the stage is written out with the destination-
// aligned copy above.  Vectors stay inside the 16-byte units that hold the first and the last source byte (same pages).
constexpr int kStageBytes = 8192;
__device__ __forceinline__ void cta_copy_from_host(uint8_t* dst, const uint8_t* src, int64_t n, uint8_t* stage /* kStageBytes + 32, 16-byte aligned */) {
  const int tid = threadIdx.x, nt = blockDim.x;
  for (int64_t o = 0; o < n; o += kStageBytes) {
    const int64_t len = n - o < kStageBytes ? n - o : kStageBytes;
    const uintptr_t a = reinterpret_cast<uintptr_t>(src + o);
    const uint4* base = reinterpret_cast<const uint4*>(a & ~static_cast<uintptr_t>(15));
    const int lead = static_cast<int>(a & 15);
    const int nvec = static_cast<int>((lead + len + 15) >> 4);
    __syncthreads();  // the previous stage has been consumed
    for (int v = tid; v < nvec; v += nt) reinterpret_cast<uint4*>(stage)[v] = base[v];
    __syncthreads();
    cta_copy(dst + o, stage + lead, len, true);
  }
}

__device__ __forceinline__ void cta_zero(uint8_t* dst, int64_t n) {
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) dst[i] = 0;
}

// grid (pieces, nreq): object bytes -> staging buffer
__global__ void __launch_bounds__(256) batch_gather_kernel(const BatchCopyParams p) {
  const BatchReqDesc& r = p.reqs[blockIdx.y];
  const int64_t full_bytes = r.len / p.bs * p.bs, tail = r.len - full_bytes;
  constexpr int64_t kPiece = 32 << 10;
  __shared__ __align__(16) uint8_t stage[kStageBytes + 32];
  for (int64_t o = static_cast<int64_t>(blockIdx.x) * kPiece; o < full_bytes; o += static_cast<int64_t>(gridDim.x) * kPiece)
    cta_copy_from_host(p.staged + r.full0 * p.bs + o, r.src + o, full_bytes - o < kPiece ? full_bytes - o : kPiece, stage);
  for (int64_t o = static_cast<int64_t>(blockIdx.x) * kPiece; o < tail; o += static_cast<int64_t>(gridDim.x) * kPiece)
    cta_copy_from_host(p.staged + r.tail_src_off + o, r.src + full_bytes + o, tail - o < kPiece ? tail - o : kPiece, stage);
}

// grid (block stride, k + m, nreq): frames (or data digests) of one drive of one request
__global__ void __launch_bounds__(128) batch_scatter_kernel(const BatchCopyParams p) {
  const BatchReqDesc& r = p.reqs[blockIdx.z];
  const int i = blockIdx.y, k = p.k, m = p.m, n = k + m;
  const int64_t nfull = r.len / p.bs, tail = r.len % p.bs, nb = nfull + (tail ? 1 : 0);
  const int64_t fstride = 32 + p.S;
  uint8_t* f = r.files[i];
  const bool frames = f != nullptr && (i >= k || r.with_data);
  const bool ddig = i < k && r.data_digests != nullptr;
  if (!frames && !ddig) return;
  for (int64_t b = blockIdx.x; b < nb; b += gridDim.x) {
    const bool is_tail = b >= nfull;
    const int64_t slot = is_tail ? r.tail_slot : r.full0 + b;
    const uint8_t* dg = p.digests + (slot * n + i) * 32;
    if (ddig) cta_copy(r.data_digests + (b * k + i) * 32, dg, 32, false);
    if (!frames) continue;
    const int64_t per = is_tail ? (tail + k - 1) / k : p.S, blen = is_tail ? tail : p.bs;
    uint8_t* fr = f + b * fstride;
    cta_copy(fr, dg, 32, false);  // hash first, then the shard (cmd/bitrot-streaming.go:60,65)
    if (i >= k) {
      cta_copy(fr + 32, p.parity + (slot * m + (i - k)) * p.pitch, per, false);
    } else {
      int64_t have = blen - static_cast<int64_t>(i) * per;
      have = have < 0 ? 0 : (have > per ? per : have);
      const uint8_t* sb = is_tail ? p.staged + r.tail_src_off : p.staged + slot * p.bs;
      if (have > 0) cta_copy(fr + 32, sb + static_cast<int64_t>(i) * per, have, false);
      if (have < per) cta_zero(fr + 32 + have, per - have);  // Split's zero padding (cmd/erasure-coding.go:81)
    }
  }
}

}  // namespace mec

// ---- degraded / plain GETs of many requests, each with its own reader set -----------------------------------------------------
namespace mec {

struct BatchGetDesc {
  const uint8_t* files[kBatchMaxFiles];  // host (mapped) part files, from their first byte; nullptr = offline
  uint8_t* dst;                          // host (mapped): object bytes [offset, offset + length)
  int64_t offset, length, total;
  int64_t start_block, nblocks;          // blocks of the part that are read
  int64_t slot0;                         // merged layout: slot of the request's first FULL block
  int64_t tail_slot;                     // slot of the part's short last block when the range reaches it, -1 otherwise
  int64_t last_len;                      // shard length of that block
  int32_t dma;                           // 1: the copy engines stage this request's frames (long ranges), the gather kernel skips it
  uint32_t whole_pos;                    // bit t: arena position t is a whole-file reader, laid by batch_whole_rows_kernel (no frames)
  // the request's decode plan (a batch of one erasure pattern: the same for every request)
  int8_t chosen[32];                     // reader set (ascending shard indices), arena position t -> shard
  int8_t targets[16];                    // rebuilt shards (GET: the data shards not read; heal: the stale drives), output row q -> shard
  int32_t r;                             // targets of this request (<= BatchGetParams::r)
  int32_t pattern;                       // its plan in the launch's pattern table
};

struct BatchGetParams {
  const BatchGetDesc* reqs;
  int nreq, k, r;                        // r: the most targets of any request (rows per slot of `rebuilt`, digests per slot k + r)
  int64_t bs, S, P;                      // block size, full shard size, device frame pitch
  uint8_t* arena;                        // survivors: reader position t at arena + t*arena_stride, slot s at + s*P
  int64_t arena_stride;
  const uint8_t* rebuilt;                // rows (slot*r + q)*pitch
  int64_t pitch;
};

__host__ __device__ __forceinline__ int64_t get_slot(const BatchGetDesc& r, int64_t b) {
  return (r.tail_slot >= 0 && b == r.nblocks - 1) ? r.tail_slot : r.slot0 + b;
}

// grid (block stride, k reader positions, nreq): frames of the chosen readers -> arena (whole-file positions have no frames)
__global__ void __launch_bounds__(128) batch_get_gather_kernel(const BatchGetParams p) {
  const BatchGetDesc& r = p.reqs[blockIdx.z];
  const int t = blockIdx.y;
  if (r.dma || ((r.whole_pos >> t) & 1)) return;
  const uint8_t* f = r.files[r.chosen[t]];
  const int64_t fstride = 32 + p.S;
  __shared__ __align__(16) uint8_t stage[kStageBytes + 32];
  for (int64_t b = blockIdx.x; b < r.nblocks; b += gridDim.x) {
    const bool is_tail = r.tail_slot >= 0 && b == r.nblocks - 1;
    const int64_t cur = is_tail ? r.last_len : p.S;
    cta_copy_from_host(p.arena + t * p.arena_stride + get_slot(r, b) * p.P, f + (r.start_block + b) * fstride, 32 + cur, stage);
  }
}

// grid (block stride, k data shards, nreq): writeDataBlocks (cmd/erasure-utils.go:42) — the wanted bytes of every data shard, read
// or rebuilt, into the caller's buffer
__global__ void __launch_bounds__(128) batch_get_scatter_kernel(const BatchGetParams p) {
  const BatchGetDesc& r = p.reqs[blockIdx.z];
  const int i = blockIdx.y;
  int t = -1, q = -1;
  for (int x = 0; x < p.k; x++) if (r.chosen[x] == i) t = x;
  for (int x = 0; x < r.r; x++) if (r.targets[x] == i) q = x;
  if (t < 0 && q < 0) return;
  const int64_t hi = r.offset + r.length;
  for (int64_t b = blockIdx.x; b < r.nblocks; b += gridDim.x) {
    const bool is_tail = r.tail_slot >= 0 && b == r.nblocks - 1;
    const int64_t cur = is_tail ? r.last_len : p.S, slot = get_slot(r, b);
    const int64_t B = r.start_block + b, blo = B * p.bs, bhi = blo + p.bs < r.total ? blo + p.bs : r.total;
    const int64_t slo = blo + static_cast<int64_t>(i) * cur, shi = slo + cur < bhi ? slo + cur : bhi;
    const int64_t a = slo > r.offset ? slo : r.offset, e = shi < hi ? shi : hi;
    if (e <= a) continue;
    const uint8_t* src = t >= 0 ? p.arena + t * p.arena_stride + slot * p.P + 32 : p.rebuilt + (slot * p.r + q) * p.pitch;
    cta_copy(r.dst + (a - r.offset), src + (a - slo), e - a, false);
  }
}

// grid (block stride, r rebuilt shards, nreq): healed frames of every stale drive of every request — multiWriter{writeQuorum: 1} +
// streamingBitrotWriter.Write (cmd/erasure-decode.go:317-366, cmd/bitrot-streaming.go:57-69): [digest of the rebuilt shard][shard]
// at frame b of outs[req * r + q] (r = the batch's most stale drives, q < the request's own), the part's short last frame 32 + last_len bytes.  Digests [slot][k + r][32] (outputs behind
// the k inputs), rebuilt rows (slot * r + q) * pitch.  Nothing outside a frame is written.
__global__ void __launch_bounds__(128) batch_heal_scatter_kernel(const BatchGetParams p, const uint8_t* digests, uint8_t* const* outs) {
  const BatchGetDesc& r = p.reqs[blockIdx.z];
  const int q = blockIdx.y;
  if (q >= r.r) return;
  uint8_t* f = outs[static_cast<int64_t>(blockIdx.z) * p.r + q];
  const int64_t fstride = 32 + p.S;
  for (int64_t b = blockIdx.x; b < r.nblocks; b += gridDim.x) {
    const bool is_tail = r.tail_slot >= 0 && b == r.nblocks - 1;
    const int64_t slot = get_slot(r, b);
    uint8_t* fr = f + (r.start_block + b) * fstride;
    cta_copy(fr, digests + (slot * (p.k + p.r) + p.k + q) * 32, 32, false);  // hash first, then the shard
    cta_copy(fr + 32, p.rebuilt + (slot * p.r + q) * p.pitch, is_tail ? r.last_len : p.S, false);
  }
}

}  // namespace mec

// ---- data movement between pools (mec_transcode): the data shards of a reconstructed chunk -> its contiguous object bytes -------
namespace mec {

struct ResplitParams {
  uint8_t* obj;                 // device: object bytes of the chunk's blocks, block b at b*bs (the short last block right behind the full ones)
  const uint8_t* arena;         // survivors: reader position t at arena + t*arena_stride, block b's frame at + b*P (shard at + 32)
  int64_t arena_stride, P;
  const uint8_t* rebuilt;       // rebuilt data shards: block b, row q at (b*r + q)*pitch
  int64_t pitch;
  int64_t bs, S;                // block size, full shard length
  int64_t nfull;                // full blocks of the chunk
  int64_t tail, tail_S;         // object bytes and shard length of the part's short last block behind them (tail 0: none)
  int r;
  int8_t src[kBatchMaxFiles];   // data shard i: read at arena position src[i] >= 0, or rebuilt row -1 - src[i]
};

// grid (blocks of the chunk, k source data shards), 128 threads: writeDataBlocks (cmd/erasure-utils.go:42) into device memory.
// CTA (b, i) copies the object bytes of data shard i of block b, never Split's zero padding, to obj + b*bs + i*S_b.  Sources are
// 16-byte aligned rows; destinations land at any offset (S = 87382 for RS(12,4)), so cta_copy stores destination-aligned 16-byte
// vectors from a funnel-shifted source.  It reads up to one word past a row: inside the arena's 512-byte padding, and inside the
// slack DevBuf keeps behind every rebuilt-row buffer (at least 256 bytes) for the chunk's last row, which ends at round_up(S, 16).
// __grid_constant__: src[i] is read straight from the parameter bank (a by-value parameter indexed at run time is copied to the stack).
__global__ void __launch_bounds__(128) transcode_resplit_kernel(const __grid_constant__ ResplitParams p) {
  const int64_t b = blockIdx.x;
  const int i = blockIdx.y;
  const bool is_tail = b >= p.nfull;
  const int64_t per = is_tail ? p.tail_S : p.S, blen = is_tail ? p.tail : p.bs;
  int64_t have = blen - static_cast<int64_t>(i) * per;
  have = have < 0 ? 0 : (have > per ? per : have);
  if (have == 0) return;
  const int t = p.src[i];
  const uint8_t* src = t >= 0 ? p.arena + t * p.arena_stride + b * p.P + 32 : p.rebuilt + (b * p.r + (-1 - t)) * p.pitch;
  cta_copy(p.obj + b * p.bs + static_cast<int64_t>(i) * per, src, have, false);
}

// ---- mec_transcode_whole: a part of a whole-file bitrot algorithm has no frames; its verified shard files sit raw on the device ----
struct WholeResplitParams {
  uint8_t* obj;                 // device: object bytes of the chunk's source blocks, chunk block b at b*bs
  const uint8_t* arena;         // verified raw shard files: arena position t at arena + t*fpitch, part block B's shard at + B*S
  int64_t fpitch;               // >= round_up(shard file size, 16) + 256 (the padding the copy may read into)
  const uint8_t* rebuilt;       // rebuilt data shards of the chunk: chunk block b, row q at (b*r + q)*pitch
  int64_t pitch;
  int64_t b0;                   // part block of the chunk's first block
  int64_t bs, S, total;         // source block size, full shard length, part length
  int k, r;
  int8_t src[kBatchMaxFiles];   // data shard i: read at arena position src[i] >= 0, or rebuilt row -1 - src[i]
};

// grid (source blocks of the chunk, k source data shards), 128 threads: writeDataBlocks (cmd/erasure-utils.go:42) into device
// memory.  CTA (b, i) copies the object bytes of data shard i of part block B = b0 + b to obj + b*bs + i*S_B, where S_B =
// ceil(blen / k) and blen = min(bs, total - B*bs): the byte count comes from the part length, so Split's zero padding is never
// copied, even when the short last block's shards are S long.  Raw shards lie at B*S inside a shard file, any byte offset (S =
// 87382 for RS(12,4) at 1 MiB), and land at any offset: cta_copy stores destination-aligned 16-byte vectors built from 4-byte
// loads and funnel shifts, reading at most one word past a shard, which stays inside a file's 256 bytes of padding and inside
// the 256 bytes the caller allocates behind the last rebuilt row.
__global__ void __launch_bounds__(128) whole_resplit_kernel(const __grid_constant__ WholeResplitParams p) {
  const int64_t b = blockIdx.x, B = p.b0 + b;
  const int i = blockIdx.y;
  const int64_t blen = p.total - B * p.bs < p.bs ? p.total - B * p.bs : p.bs;
  const int64_t per = (blen + p.k - 1) / p.k;
  int64_t have = blen - static_cast<int64_t>(i) * per;
  have = have < 0 ? 0 : (have > per ? per : have);
  if (have == 0) return;
  const int t = p.src[i];
  const uint8_t* src = t >= 0 ? p.arena + t * p.fpitch + B * p.S : p.rebuilt + (b * p.r + (-1 - t)) * p.pitch;
  cta_copy(p.obj + b * p.bs + static_cast<int64_t>(i) * per, src, have, false);
}

// grid (block stride, k source data shards, nreq), 128 threads: the batched form of transcode_resplit_kernel for a merged batch of
// moves (mec_batcher_transcode).  Request z's decode plan (chosen readers, rebuilt data shards) and its source slots come from the
// read table p.reqs[z], which covers the whole part (start_block 0); where its object bytes go comes from the PUT table d.reqs[z]
// (len = total): full destination blocks at d.staged + full0 * d.bs onwards, the short last destination block at d.staged +
// tail_src_off.  CTA (x, i, z) copies the object bytes of data shard i of every source block of request z, never Split's zero
// padding.  Source block b (source block size p.bs) holds object bytes [b * p.bs, (b + 1) * p.bs); the destination block size d.bs
// divides p.bs, so those bytes are whole destination blocks, except at the end of the part.  A shard's run of object bytes
// [o, o + have) lies in the contiguous full destination blocks below edge = (len / d.bs) * d.bs and in the short last destination
// block above it; a run that straddles the edge is copied in two pieces.  The source's short last slot (shard length last_len) may
// still hold a short object block when ceil(tail / k) == S, so each block's byte count is taken from the part length.  Source rows
// are read up to one word past their end, inside the arena's padding and the slack behind the rebuilt rows (see
// transcode_resplit_kernel).
__global__ void __launch_bounds__(128) batch_transcode_resplit_kernel(const BatchGetParams p, const BatchCopyParams d) {
  const BatchGetDesc& r = p.reqs[blockIdx.z];
  const BatchReqDesc& w = d.reqs[blockIdx.z];
  const int i = blockIdx.y;
  int t = -1, q = -1;
  for (int x = 0; x < p.k; x++) if (r.chosen[x] == i) t = x;
  for (int x = 0; x < r.r; x++) if (r.targets[x] == i) q = x;
  if (t < 0 && q < 0) return;
  const int64_t edge = w.len / d.bs * d.bs;
  uint8_t* const full = d.staged + w.full0 * d.bs;
  for (int64_t b = blockIdx.x; b < r.nblocks; b += gridDim.x) {
    const bool is_tail = r.tail_slot >= 0 && b == r.nblocks - 1;
    const int64_t cur = is_tail ? r.last_len : p.S, slot = get_slot(r, b);
    const int64_t blen = w.len - b * p.bs < p.bs ? w.len - b * p.bs : p.bs;
    int64_t have = blen - static_cast<int64_t>(i) * cur;
    have = have > cur ? cur : have;
    if (have <= 0) continue;
    const uint8_t* src = t >= 0 ? p.arena + t * p.arena_stride + slot * p.P + 32 : p.rebuilt + (slot * p.r + q) * p.pitch;
    const int64_t o = b * p.bs + static_cast<int64_t>(i) * cur;
    const int64_t lo = o < edge ? (edge - o < have ? edge - o : have) : 0;  // bytes below the edge
    if (lo > 0) cta_copy(full + o, src, lo, false);
    if (lo < have) cta_copy(d.staged + w.tail_src_off + (o + lo - edge), src + lo, have - lo, false);
  }
}

// grid (block stride, k reader positions, nreq), 128 threads: the whole-file readers of a merged batch — every reader of a whole-file
// move (mec_batcher_transcode_whole), the whole-file readers of a mixed GET or heal (mec_batcher_decode_mixed / _heal_mixed).  Their
// raw shard files sit in a device file arena, one stream-table entry per whole-file reader: position t of request z (bit t of
// whole_pos) is stream first[z] + (whole-file positions of z below t), its file at files + streams[that].off (16-byte aligned, at
// least 256 readable bytes behind it), block b's shard at + b * S.  This lays every such shard into the frame arena slot a GET batch
// would have staged it in (shard at + 32, the digest bytes are left as they are), so the merged reconstruct, the scatters and
// batch_transcode_resplit_kernel run on it unchanged.  Other positions are left to the frame staging.  Sources sit at any byte
// offset (S = 87382 for RS(12,4) at 1 MiB); cta_copy reads at most one word past a shard, inside the file's padding.
__global__ void __launch_bounds__(128) batch_whole_rows_kernel(const BatchGetParams p, const uint8_t* files, const WholeStream* streams,
                                                               const int32_t* first) {
  const BatchGetDesc& r = p.reqs[blockIdx.z];
  const int t = blockIdx.y;
  if (!((r.whole_pos >> t) & 1)) return;
  const uint8_t* f = files + streams[first[blockIdx.z] + __popc(r.whole_pos & ((1u << t) - 1))].off;
  for (int64_t b = blockIdx.x; b < r.nblocks; b += gridDim.x) {
    const bool is_tail = r.tail_slot >= 0 && b == r.nblocks - 1;
    cta_copy(p.arena + t * p.arena_stride + get_slot(r, b) * p.P + 32, f + (r.start_block + b) * p.S, is_tail ? r.last_len : p.S, false);
  }
}

// ---- mec_decode_mixed / mec_heal_mixed: whole-file readers beside streaming ones in the reconstruct pipeline --------------------
struct WholeFramesParams {
  uint8_t* arena;               // chunk arena: reader position t at arena + t*arena_stride, chunk block b's frame at + b*P
  int64_t arena_stride, P;
  const uint8_t* files;         // verified raw shard files: file slot f at files + f*fpitch (at least 256 readable bytes behind it)
  int64_t fpitch;
  int64_t S, first;             // full shard length; file block of the chunk's first block
  int64_t nb, last_len;         // blocks of the chunk; shard length of its last block
  int ncols;                    // whole-file positions of the chunk
  int8_t pos[kBatchMaxFiles];   // column y: arena position pos[y], file slot file[y]
  int8_t file[kBatchMaxFiles];
};

// grid (blocks of the chunk, whole-file positions), 128 threads: the single-request form of batch_whole_rows_kernel.  CTA (b, y)
// lays row first + b of file file[y] into frame slot b of arena position pos[y] (shard at + 32; the digest bytes are left as they
// are, the reconstruct does not check them), so the fused reconstruct and both sinks run on the chunk arena unchanged.  Rows sit
// at any byte offset (S = 87382 for RS(12,4) at 1 MiB, 873814 at 10 MiB); cta_copy reads at most one word past a row, inside the
// file's padding for its last row.
__global__ void __launch_bounds__(128) whole_rows_frames_kernel(const __grid_constant__ WholeFramesParams p) {
  const int64_t b = blockIdx.x;
  const int y = blockIdx.y;
  const uint8_t* row = p.files + p.file[y] * p.fpitch + (p.first + b) * p.S;
  cta_copy(p.arena + p.pos[y] * p.arena_stride + b * p.P + 32, row, b == p.nb - 1 ? p.last_len : p.S, false);
}

}  // namespace mec
