// ec_kernel.cuh — the fused Reed-Solomon + HighwayHash-256 kernel (sm_90a).
//
// One launch consumes `nblocks` erasure blocks.  For each block it reads k input shards ONCE
// (cmd/erasure-coding.go:81 Split layout for encode; surviving shards for reconstruct/heal),
// produces r output shards (parity rows of cmd/erasure-coding.go:85, or the decode rows behind
// :106/:112) and the HighwayHash-256 bitrot digest of every input and output shard
// (cmd/bitrot-streaming.go:57-59 for writers, :194-196 for readers) — the two passes the
// reference makes over each shard are one pass over shared-memory tiles here.
//
// Work decomposition (all integer/byte work, ALU-issue- and HBM-bound; no tensor cores):
//   CTA      = `eb` erasure blocks (4 in the specialised kernels: one warp per block), blockDim = 2*(k+r)*eb rounded
//              up to a warp multiple; persistent grid of as many CTAs as fit (7 per SM for RS(12,4); the misaligned 3-D encode launches
//              as many as a budget of load bytes in flight allows, 5 per SM for RS(12,4))
//   tile     = 256 bytes of every shard.  Shards start at arbitrary byte offsets of the object
//              (S = ceil(blockSize/k) is 87382 for RS(12,4)@1MiB) but TMA boxes must start on 16-byte boundaries
//              (tools/tma_probe.cu), so each row is fetched as a 16B-aligned superset ("raw" tile, cp.async.bulk.tensor
//              with u32 elements: 3-D requests of several rows x eb blocks at a 288-byte pitch for the specialised
//              encode, one 272-byte 2-D box per row otherwise; Split's zero padding = TMA out-of-bounds fill)
//   GF step  = each thread owns an 8-byte column: rows are re-aligned in registers (PRMT with compile-time selectors when
//              S mod 16 is a template constant), re-stored into the "aligned" tile for the hash threads, and multiplied
//              -> r outputs -> STS.64 + STG.64
//   HH step  = two threads per shard stream (64-bit lanes {0,1} / {2,3}); rows of the aligned tile have a 288-byte pitch
//              so the four streams of a quarter-warp hit disjoint banks
//   pipeline = raw tile i+1 is in flight (TMA) while the hash threads chew on aligned tile i; two CTA barriers per tile
//   direct   = inputs whose rows are all 16-byte aligned (reconstruct / heal / verify frames, encode with S mod 16 == 0)
//              skip the raw -> aligned copy: TMA writes the 288-byte-pitch rows the hash threads read, two buffers
//              alternate, tile i+2 is requested as soon as tile i is consumed
#pragma once
#include "ec_device.cuh"

namespace mec {

constexpr int kTile = 256;       // bytes of one shard per tile
constexpr int kRawRow = 272;     // 16B-aligned superset of a tile row
constexpr int kRowPitch = 288;   // pitch of the aligned data / output tiles (bank skew of 32 B)
constexpr int kMaxK = 32;        // inputs supported by the GPU path
constexpr int kMaxR = 16;        // outputs supported by the GPU path
constexpr int kMaxMaps = 16;     // tensor maps carried in kernel params
constexpr int kRChunk = 4;       // widest row chunk of the runtime-matrix GF step (mask table padding)
constexpr int kAlignRuntime = -1;

#ifndef MEC_PHASE_CYCLES
#define MEC_PHASE_CYCLES 0  // 1: per-phase cycle counters in the throughput kernel (PhaseSlot below); never in a shipped build
#endif

enum LoaderMode : int { kLoadBytewise = 0, kLoadTmaBlocks2D = 1, kLoadTmaPerInput = 2, kLoadTmaRuns = 3 };
constexpr int kMaxRuns = 6;      // runs of uniformly spaced input rows fetched with one 3-D request each (kLoadTmaRuns)

struct alignas(64) TmaMaps {
  CUtensorMap m[kMaxMaps];
};

// latency kernel, contiguous encode: the geometry of every erasure block of a launch — blocks of different objects (full blocks and the
// short last blocks of many PutObjects) ride in ONE launch
struct SmallBlock {
  int64_t in_off;   // bytes from FusedParams::in_ptr[0] to the block's first byte; row t starts S * t further on
  int32_t S;        // shard bytes of this block = ceil(bytes / k)
  int32_t bytes;    // object bytes in the block (Split pads the rest of k * S with zeros)
};

// latency kernel, runtime matrix: the decode plan of one erasure pattern — reads of many objects whose shard indices are rotated
// differently (hashOrder, cmd/erasure-metadata-utils.go:178) ride in ONE launch, each block with its own matrix
struct SmallPattern {
  int32_t r;                     // rows this pattern rebuilds (<= the launch's r); 0: hash and verify only
  uint8_t coef[kMaxR][kMaxK];    // r x k decode rows
};

struct FusedParams {
  int k, r, eb, tma_mode;
  int tiles_3d;                    // ROWS3D: tiles [0, tiles_3d) of a shard are fetched with one 3-D request
  int raw_pitch;                   // bytes between erasure blocks inside a raw row group (272; 384 when every row is its own TMA box)
  int64_t nblocks;
  int nhash;                       // streams hashed per erasure block: k + r, or k when the outputs carry no digest
  int32_t S;                       // shard bytes per erasure block
  int32_t in_c0_block_step;        // kLoadTmaPerInput: bytes between blocks in an input stream (multiple of 16)
  int32_t in_c0[kMaxK];            // TMA: 16B-aligned byte coordinate of input t (block 0, x = 0)
  uint8_t in_align[kMaxK];         // TMA: bytes to skip at the start of each raw row (0..15)
  const uint8_t* in_ptr[kMaxK];    // byte-wise loader: input t, block 0, x = 0
  int64_t in_block_stride;         // byte-wise loader: bytes between blocks
  int64_t in_limit, in_shard_step; // valid bytes of input t = clamp(in_limit - t*in_shard_step, 0, S)
  uint8_t* out;                    // output shard (b, j) at out + (b*r + j) * out_pitch
  int64_t out_pitch;               // multiple of 16
  uint8_t* digests;                // [nblocks][k + r][32]; nullptr = no hashing
  const uint8_t* expect_ptr[kMaxK];// optional expected digest of input t, block 0 (bitrot reader)
  int64_t expect_block_stride;
  uint8_t* corrupt;                // optional [nblocks][k], set to 1 on digest mismatch
  uint64_t key[4];                 // HighwayHash key (cmd/bitrot.go:37 for bitrot)
  uint8_t coef[kMaxR][kMaxK];      // runtime matrix (GfDynamic only)
  int32_t nruns;                   // kLoadTmaRuns: input rows [run_row0[q], run_row0[q+1]) share tensor map q (x, block, row)
  uint8_t run_row0[kMaxRuns + 1];
  uint32_t* work_counter;          // optional: groups beyond the first of every CTA are claimed from this counter (zeroed per launch)
  const int32_t* block_len;        // latency kernel only: shard bytes of every erasure block (nullptr: S for all) — frames of many files in one launch
  const SmallBlock* blocks;        // latency kernel only, contiguous encode: per-block offset / shard bytes / object bytes (nullptr: uniform)
  const SmallPattern* patterns;    // latency kernel only, runtime matrix: decode plans of the launch (nullptr: coef / r for all blocks)
  const uint16_t* block_pattern;   // ... and the index of every block's plan in `patterns`
  // latency kernel only: ONE block of the launch (an object's short last block) differs from the rest — no table needed
  int64_t tail_block;              // its index, -1 = none
  int64_t tail_in_off;             // contiguous encode: bytes from in_ptr[0] to its first byte (rows S_tail apart); -1: rows addressed like the others
  int32_t tail_S, tail_bytes;      // its shard bytes; contiguous encode: its object bytes
#if MEC_PHASE_CYCLES
  unsigned long long* phase;       // cycle attribution counters (layout at PhaseSlot), nullptr = off
#endif
};

#if MEC_PHASE_CYCLES
// Cycle attribution of the throughput kernel (build with -DMEC_PHASE_CYCLES=1; tools/phase_cycles.py reads it).  Lane 0 of
// every warp adds the SM-clock cycles its warp spent in each phase of a tile to counters of its SM (one 64-byte line per SM,
// so the adds of different SMs do not meet in L2).  Warp 0 of every CTA also adds its CTA's lifetime in SM cycles and in
// %globaltimer nanoseconds, which gives the clock the SM really ran at; slots 0 / 1 take the earliest start and latest end
// of the launch in %globaltimer ns.  Counters start at phase + kPhaseHeader + 8 * smid.
enum PhaseSlot : int { kPhTma = 0, kPhBarA, kPhBarB, kPhGf, kPhHh, kPhWarp, kPhCtaClk, kPhCtaNs };
constexpr int kPhaseHeader = 8, kPhaseMaxSm = 256;
__device__ __forceinline__ uint32_t clock32() {
  uint32_t c;
  asm volatile("mov.u32 %0, %%clock;" : "=r"(c) :: "memory");
  return c;
}
__device__ __forceinline__ uint64_t clock64v() {
  uint64_t c;
  asm volatile("mov.u64 %0, %%clock64;" : "=l"(c) :: "memory");
  return c;
}
__device__ __forceinline__ uint64_t global_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t) :: "memory");
  return t;
}
__device__ __forceinline__ unsigned long long* phase_sm(unsigned long long* phase) {
  uint32_t smid;
  asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
  return phase + kPhaseHeader + 8 * (smid % kPhaseMaxSm);
}
// lap(slot): the cycles since the previous lap go to `slot`.  Only the 32-bit time stamp stays live across a tile, so the
// instrumented kernel keeps the register budget (and the occupancy) of the shipped one.
struct PhaseTimer {
  unsigned long long* phase;
  uint32_t t;
  __device__ __forceinline__ void lap(int slot) {
    const uint32_t n = clock32();
    if (phase != nullptr && (threadIdx.x & 31) == 0) atomicAdd(phase_sm(phase) + slot, static_cast<unsigned long long>(n - t));
    t = n;
  }
  // start / end of an interval added to a 64-bit slot as (end - start): one add each, nothing held in registers
  __device__ __forceinline__ void open64(int slot, uint64_t now) const { if (phase != nullptr) atomicAdd(phase_sm(phase) + slot, 0ull - now); }
  __device__ __forceinline__ void close64(int slot, uint64_t now) const { if (phase != nullptr) atomicAdd(phase_sm(phase) + slot, static_cast<unsigned long long>(now)); }
};
#define MEC_PHASE(slot) ph.lap(slot)
#define MEC_PHASE_SKIP() (ph.t = clock32())
#else
#define MEC_PHASE(slot) ((void)0)
#define MEC_PHASE_SKIP() ((void)0)
#endif

// ------------------------------------------------------------------ GF policies
template <int K_, int M_>
struct GfStatic {
  static constexpr bool kIsStatic = true;
  static constexpr int K = K_, R = M_;
  static constexpr int kHashOut = 1;  // outputs always carry a digest (encode)
  using Mat = EncodeMatrix<K_, M_>;
};
template <int RC_>  // rows of the runtime matrix handled per pass over the inputs (1, 2 or 4)
struct GfDynamic {
  static constexpr bool kIsStatic = false;
  static constexpr int K = 0, R = 0, RC = RC_;
  static constexpr int kHashOut = -1;  // FusedParams::nhash decides at run time
};

__host__ __device__ constexpr uint32_t raw_group_bytes(int eb, int raw_pitch) { return (static_cast<uint32_t>(eb) * raw_pitch + 127u) & ~127u; }

// `direct`: every input row is 16-byte aligned, TMA writes straight into the 288-byte-pitch rows the hash threads read —
// two such buffers (tile i is hashed while tile i+1 lands), no re-aligned copy.  Otherwise: one raw tile + one aligned tile.
// raw_rows: rows of the raw tile when the 3-D fetch needs more than k of them (raw_rows_3d); 0 = k
__host__ __device__ constexpr uint32_t fused_smem_bytes(int k, int r, int eb, int raw_pitch, bool dynamic_gf, bool direct = false,
                                                        int raw_rows = 0) {
  uint32_t b = 0;  // the mbarriers live in row padding; the dynamic segment is declared 128-byte aligned
  if (direct) {
    b += static_cast<uint32_t>(2 * k + (r > 0 ? r : 0)) * raw_group_bytes(eb, kRowPitch);
    if (r <= 0) b += 128;  // no output rows to hide the barriers in
  } else {
    b += static_cast<uint32_t>(raw_rows > k ? raw_rows : k) * raw_group_bytes(eb, raw_pitch);
    b += static_cast<uint32_t>(k + (r > 0 ? r : 0)) * eb * kRowPitch;
  }
  if (dynamic_gf) b += static_cast<uint32_t>(k) * ((r + kRChunk - 1) / kRChunk) * kRChunk * 8 * 4;
  return b;
}
__host__ __device__ constexpr bool fused_is_direct(bool use_tma, int align, bool autop) { return use_tma && align == 0 && !autop; }

// 3-D fetch mode: the k shard rows of a tile arrive in ceil(k / RG) requests of RG consecutive rows x eb blocks.  Inside
// the tensor map every row sits at the uniform stride S & ~15, so row t starts t * (S mod 16) bytes into "its" map row;
// each request starts at the 16-byte boundary below its first row, which leaves row t with row_lead_3d() leading bytes.
// RG is the largest group whose widest row still fits the 288-byte pitch of the aligned tile: one request for shards
// that are 16-byte multiples, three for RS(12,4) at 1 MiB (S mod 16 = 6) — the narrow pitch is what lets a seventh CTA
// fit on the SM.
__host__ __device__ constexpr int group_shift_3d(int g, int sm16, int rg) { return (g * rg * sm16) & ~15; }
__host__ __device__ constexpr int row_lead_3d(int t, int sm16, int rg) { return t * sm16 - group_shift_3d(t / rg, sm16, rg); }
__host__ __device__ constexpr int raw_row_3d(int k, int sm16, int eb, int rg) {
  int lead = 0;
  for (int t = 0; t < k; t++) lead = row_lead_3d(t, sm16, rg) > lead ? row_lead_3d(t, sm16, rg) : lead;
  int r = (kTile + lead + 15) / 16 * 16;
  while ((rg * eb * r) % 128) r += 16;  // every request lands on a 128-byte boundary
  return r;
}
__host__ __device__ constexpr int rows_per_request_3d(int k, int sm16, int eb) {
  for (int rg = k; rg > 1; rg--)
    if (raw_row_3d(k, sm16, eb, rg) <= kRowPitch && (eb * raw_row_3d(k, sm16, eb, rg)) % 128 == 0) return rg;
  return 1;
}
__host__ __device__ constexpr int raw_row_3d(int k, int sm16, int eb) { return raw_row_3d(k, sm16, eb, rows_per_request_3d(k, sm16, eb)); }
// Rows of the raw tile with the 3-D fetch.  The last request of a tile lands RG whole rows even when fewer than RG shard rows are
// left (those past k are out of bounds of the tensor map and arrive zero-filled), so the raw tile holds k rounded up to a multiple
// of RG rows — RS(10,4) with S mod 16 = 5 takes two requests of seven rows.  Every compiled geometry has k % RG == 0.
__host__ __device__ constexpr int raw_rows_3d(int k, int rg) { return (k + rg - 1) / rg * rg; }
static_assert(raw_rows_3d(12, rows_per_request_3d(12, 6, 4)) == 12 && raw_rows_3d(6, rows_per_request_3d(6, 11, 4)) == 6 &&
                  raw_rows_3d(10, rows_per_request_3d(10, 5, 4)) == 14, "raw tile rows of the 3-D fetch");

// RS(12,4) at 1 MiB blocks (S mod 16 = 6): three requests of four rows at a 288-byte pitch, 32 256 bytes per CTA — seven
// CTAs (7 x (32 256 + 1 024 reserved) <= 233 472) and 28 warps x 32 lanes x 72 registers = the whole register file.
static_assert(rows_per_request_3d(12, 6, 4) == 4 && raw_row_3d(12, 6, 4) == kRowPitch, "RS(12,4) row groups");
static_assert(row_lead_3d(7, 6, 4) == 26 && row_lead_3d(8, 6, 4) == 0 && group_shift_3d(2, 6, 4) == 48, "row leads");
static_assert(fused_smem_bytes(12, 4, 4, raw_row_3d(12, 6, 4), false) == 32256, "RS(12,4) CTA footprint");
static_assert(7 * (fused_smem_bytes(12, 4, 4, raw_row_3d(12, 6, 4), false) + 1024) <= 233472, "seven CTAs per SM");
static_assert(fused_smem_bytes(12, 4, 4, kRowPitch, false, true) == 32256, "direct-fetch footprint equals raw + aligned");
static_assert(rows_per_request_3d(8, 0, 4) == 8 && raw_row_3d(8, 0, 4) == kTile, "aligned shards: one request, no padding");

#ifndef MEC_MIN_BLOCKS
#define MEC_MIN_BLOCKS 3
#endif

// one 8-byte column of raw row `row` whose logical byte 0 sits `A` bytes into the row
template <int A>
__device__ __forceinline__ uint2 load_col_ct(const uint8_t* row) {
  constexpr int base = A & ~3, sh = A & 3;
  if constexpr (sh == 0 && (base & 7) == 0) {
    return *reinterpret_cast<const uint2*>(row + base);
  } else if constexpr (sh == 0) {
    const uint32_t* w = reinterpret_cast<const uint32_t*>(row + base);
    return make_uint2(w[0], w[1]);
  } else {
    const uint32_t* w = reinterpret_cast<const uint32_t*>(row + base);
    constexpr uint32_t sel = 0x3210u + 0x1111u * sh;
    const uint32_t w0 = w[0], w1 = w[1], w2 = w[2];
    return make_uint2(prmt(w0, w1, sel), prmt(w1, w2, sel));
  }
}
__device__ __forceinline__ uint2 load_col_rt(const uint8_t* row, uint32_t a) {
  const uint32_t* w = reinterpret_cast<const uint32_t*>(row + (a & ~3u));
  const uint32_t sel = 0x3210u + 0x1111u * (a & 3u);
  const uint32_t w0 = w[0], w1 = w[1], w2 = w[2];
  return make_uint2(prmt(w0, w1, sel), prmt(w1, w2, sel));
}

// USE_TMA: tile loader.  ALIGN: S mod 16 of a contiguous (Split) input when known at compile time
// (0 = every row 16B-aligned), kAlignRuntime = per-row table in the params.  EB_T: erasure blocks
// per CTA when fixed at compile time (0 = runtime).  AUTO: k + r == 16, i.e. one warp owns exactly
// one erasure block (32 columns, 16 streams x 2 hash threads): the GF -> HH hand-off is then
// warp-local (__syncwarp) and the only CTA-wide event is "raw tile consumed": every warp arrives on a
// plain mbarrier as soon as its lanes hold their columns in registers, and the TMA-issuing lane of warp 0
// waits for that phase before it requests the next tile — no __syncthreads in the steady state.
// ROWS3D: all k rows x eb blocks of a tile arrive with ONE 3-D TMA request (x, block, row) instead of k requests;
// only the last tiles of a shard, whose box would cross the row stride, fall back to per-row requests (which also
// provide Split's zero padding through out-of-bounds fill).  Needs a compile-time ALIGN and EB_T.
// Launch bounds: with a compile-time CTA shape the register budget follows the CTAs that fit anyway — 72 registers
// when seven 128-thread CTAs fit in shared memory, 80 when shared memory stops at six.  Left alone, ptxas / NVRTC
// drift between 72 and 80 registers from one build to the next and lose a CTA per SM.
template <class GF, int EB_T>
__host__ __device__ constexpr int fused_max_threads() {
  return (EB_T > 0 && GF::K > 0) ? ((2 * (GF::K + GF::R) * EB_T + 31) / 32 * 32) : 256;
}
template <class GF, int ALIGN, int EB_T, bool ROWS3D, bool DIRECT>
__host__ __device__ constexpr int fused_min_blocks() {
  if constexpr (!GF::kIsStatic) return GF::RC >= 2 ? 2 : MEC_MIN_BLOCKS;  // 8 bit-plane accumulators per output row: two or four rows spill at 80 registers
  if (!(EB_T > 0 && GF::K > 0)) return MEC_MIN_BLOCKS;
  constexpr int t = fused_max_threads<GF, EB_T>();
  const int by_regs = 65536 / (72 * t);
  const int raw = ROWS3D ? raw_row_3d(GF::K > 0 ? GF::K : 1, ALIGN > 0 ? ALIGN : 0, EB_T > 0 ? EB_T : 1) : kRawRow;
  const int rows = ROWS3D ? raw_rows_3d(GF::K, rows_per_request_3d(GF::K > 0 ? GF::K : 1, ALIGN > 0 ? ALIGN : 0, EB_T > 0 ? EB_T : 1)) : 0;
  const int by_smem = 233472 / (static_cast<int>(fused_smem_bytes(GF::K, GF::R, EB_T, raw, false, DIRECT, rows)) + 1024);
  const int b = by_regs < by_smem ? by_regs : by_smem;
  return b > 0 ? b : 1;
}
template <class GF, bool USE_TMA, int ALIGN, int EB_T, int AUTO_MODE, bool ROWS3D = false>
__global__ void __launch_bounds__((fused_max_threads<GF, EB_T>()), (fused_min_blocks<GF, ALIGN, EB_T, ROWS3D, fused_is_direct(USE_TMA, ALIGN, AUTO_MODE == 1)>())) fused_rs_hh_kernel(const __grid_constant__ FusedParams p,
                                                                         const __grid_constant__ TmaMaps maps) {
  extern __shared__ __align__(128) uint8_t smem[];
  const int k = GF::kIsStatic ? GF::K : p.k;
  const int r = GF::kIsStatic ? GF::R : p.r;
  const int eb = EB_T > 0 ? EB_T : p.eb;
  const int nstreams = k + r;
  const int tid = threadIdx.x, nthr = blockDim.x;
  const int warp_id = __shfl_sync(0xffffffffu, tid >> 5, 0);  // provably warp-uniform
  const bool warp0 = warp_id == 0;
  // AUTO_MODE 1: warp-autonomous pipeline (no CTA barrier); 2: barrier (A) kept, barrier (B) warp-local (k + r == 16, !DIRECT)
  constexpr bool AUTO = AUTO_MODE == 1;
  constexpr bool DIRECT = fused_is_direct(USE_TMA, ALIGN, AUTO);
  constexpr bool WARP_B = AUTO_MODE == 2 && !DIRECT && USE_TMA;
  static_assert(AUTO_MODE == 0 || GF::kIsStatic, "warp-local hand-offs need one warp per erasure block: compile-time (k, r) with k + r == 16");
  constexpr int kK3 = GF::K > 0 ? GF::K : 1, kSm3 = ALIGN > 0 ? ALIGN : 0, kEb3 = EB_T > 0 ? EB_T : 1;
  constexpr int kRG = ROWS3D ? (DIRECT ? kK3 : rows_per_request_3d(kK3, kSm3, kEb3)) : 1;  // shard rows per 3-D request
  constexpr int kRaw3 = ROWS3D ? (DIRECT ? kRowPitch : raw_row_3d(kK3, kSm3, kEb3)) : kRawRow;
  const uint32_t rawp = DIRECT ? static_cast<uint32_t>(kRowPitch)
                               : (ROWS3D ? static_cast<uint32_t>(kRaw3) : (EB_T > 0 ? static_cast<uint32_t>(kRawRow) : static_cast<uint32_t>(p.raw_pitch)));
  const uint32_t group_bytes = raw_group_bytes(eb, static_cast<int>(rawp));
  const uint32_t buf_bytes = static_cast<uint32_t>(ROWS3D ? raw_rows_3d(kK3, kRG) : k) * group_bytes;
  uint8_t* s_raw = smem;                                                     // [k][group]  (DIRECT: two of them)
  uint8_t* s_clean = DIRECT ? s_raw : s_raw + buf_bytes;                     // [eb][k][kRowPitch]  (not DIRECT)
  uint8_t* s_par = DIRECT ? s_raw + 2 * buf_bytes : s_clean + static_cast<uint32_t>(k) * eb * kRowPitch;
  // output rows: [eb][r][kRowPitch], DIRECT: [r][group] like the inputs
  const uint32_t par_row = DIRECT ? group_bytes : static_cast<uint32_t>(kRowPitch);
  const uint32_t par_blk = DIRECT ? static_cast<uint32_t>(kRowPitch) : static_cast<uint32_t>(r) * kRowPitch;
  uint32_t* s_masks = reinterpret_cast<uint32_t*>(s_par + (DIRECT ? static_cast<uint32_t>(r) * group_bytes + (r > 0 ? 0u : 128u)
                                                                   : static_cast<uint32_t>(r) * eb * kRowPitch));
  // bytes [256, 288) of an aligned / output row are bank-skew padding nobody reads or writes: the mbarriers sit in row 0's
  // (DIRECT input rows are written by TMA over their full pitch, so there it is the first output row, or 128 spare bytes)
  uint64_t* bars = reinterpret_cast<uint64_t*>(DIRECT ? (r > 0 ? s_par + kTile : s_par) : s_clean + kTile);
  const int rpad = (r + kRChunk - 1) / kRChunk * kRChunk;

  const int32_t S = p.S;
  const int ntiles = (S + kTile - 1) / kTile;
  const int npk = S >> 5, rem = S & 31;

  if constexpr (USE_TMA) {
    if (tid == 0) {
      mbar_init(smem_u32(&bars[0]), 1);
      if constexpr (DIRECT) mbar_init(smem_u32(&bars[1]), 1);
      if constexpr (AUTO) mbar_init(smem_u32(&bars[2]), static_cast<uint32_t>(nthr >> 5));  // "raw tile consumed": one arrival per warp
      fence_barrier_init();
    }
  }
  if constexpr (!GF::kIsStatic) {
    // expand coefficient bytes into AND-masks: s_masks[(t*rpad + j)*8 + bit]
    for (int i = tid; i < k * rpad * 8; i += nthr) {
      const int bit = i & 7, j = (i >> 3) % rpad, t = (i >> 3) / rpad;
      const uint32_t c = j < r ? p.coef[j][t] : 0u;
      s_masks[i] = 0u - ((c >> bit) & 1u);
    }
  }
  __syncthreads();
#if MEC_PHASE_CYCLES
  PhaseTimer ph{p.phase, clock32()};
  if ((tid & 31) == 0) ph.open64(kPhWarp, clock64v());
  if (tid == 0 && p.phase != nullptr) {
    const uint64_t ns = global_ns();
    atomicMin(p.phase, static_cast<unsigned long long>(ns));
    ph.open64(kPhCtaNs, ns);
    ph.open64(kPhCtaClk, clock64v());
  }
#endif

  // ---- HighwayHash thread identity: 2 threads per stream
  const int nhash = (AUTO || GF::kHashOut == 1) ? nstreams : (GF::kHashOut == 0 ? k : p.nhash);
  const bool hh_thread = p.digests != nullptr && tid < 2 * nhash * eb;
  const int sl = tid >> 1, h = tid & 1;
  // DIRECT rows are laid out [stream][block]: the four streams of a quarter-warp are then four blocks of one shard,
  // 288 bytes apart — the same bank skew the aligned tile gets from its row pitch
  const int e_hh = hh_thread ? (DIRECT ? sl % eb : sl / nhash) : 0;
  const int srow = hh_thread ? (DIRECT ? sl / eb : sl % nhash) : 0;
  const bool is_out = srow >= k;
  const uint8_t* hh_row = is_out ? s_par + static_cast<uint32_t>(srow - k) * par_row + static_cast<uint32_t>(e_hh) * par_blk
                                 : (DIRECT ? s_raw + static_cast<uint32_t>(srow) * group_bytes + static_cast<uint32_t>(e_hh) * kRowPitch
                                           : s_clean + static_cast<uint32_t>(e_hh * k + srow) * kRowPitch);
  const uint32_t hh_addr = smem_u32(hh_row) + 16u * h;
  const uint32_t hh_flip = (DIRECT && !is_out) ? buf_bytes : 0u;  // added when the tile sits in the second buffer

  // ---- GF thread identity: one 8-byte column (threads beyond eb*32 columns idle in the GF step)
  const int ncol = eb * (kTile / 8);

  const int64_t ngroups = (p.nblocks + eb - 1) / eb;
  uint32_t it = 0;  // running tile counter (mbarrier phase bookkeeping)

  // Groups are dealt dynamically when the launch brings a counter: CTA c starts with group c, every further group is claimed
  // with one atomicAdd issued at the START of the group before it (its latency hides behind a whole group of work).  With the
  // static deal (g += gridDim.x) the CTAs that own one more group than the others decide the run time — 2.47 groups per CTA for
  // the 10240-block stream leaves a third pass in which some SMs have 4 CTAs and others 3.
  uint32_t* s_next = reinterpret_cast<uint32_t*>(bars + 3);
  for (int64_t g = blockIdx.x; g < ngroups;) {
    uint32_t claimed = 0;
    if (p.work_counter != nullptr && tid == 0) claimed = atomicAdd(p.work_counter, 1u);
    const int64_t b0 = g * eb;
    const int nb = (p.nblocks - b0) < eb ? static_cast<int>(p.nblocks - b0) : eb;
    const bool hh_live = hh_thread && e_hh < nb;

    HHHalf hs;
    hh_init(hs, p.key, h);

    // ---------------- tile loader (raw tile is single-buffered: it is free as soon as GF(i) is done)
    // TMA: called by one elected lane per warp; rows are dealt round-robin over `parts` callers so no warp
    // carries the whole issue cost (part 0 also arms the mbarrier with the total byte count — complete_tx
    // arriving before expect_tx is legal, the phase cannot complete before the arrival).  Byte-wise: all threads.
    auto issue_tile_at = [&](int i, int64_t b0, int nb, int part, int parts) {
      if constexpr (USE_TMA) {
        const uint32_t sel = DIRECT ? ((it + static_cast<uint32_t>(i)) & 1u) : 0u;  // DIRECT: tiles alternate between two buffers
        const uint32_t bar = smem_u32(&bars[sel]);
        const uint32_t dst0 = smem_u32(s_raw) + sel * buf_bytes;
        if constexpr (ROWS3D) {
          constexpr int kGroups = (kK3 + kRG - 1) / kRG;
          if (i < p.tiles_3d) {  // kGroups requests for the whole tile (rows past k are out of bounds: zero-filled into the raw tile's
                                 // spare rows, raw_rows_3d, and still counted)
            if (part == 0) {
              mbar_expect_tx(bar, static_cast<uint32_t>(kGroups * kRG) * eb * kRaw3);
#pragma unroll
              for (int gq = 0; gq < kGroups; gq++)
                tma_load_3d(dst0 + static_cast<uint32_t>(gq * kRG) * group_bytes, &maps.m[1],
                            i * (kTile / 4) + group_shift_3d(gq, kSm3, kRG) / 4, static_cast<int32_t>(b0), gq * kRG, bar);
              // No L2 prefetch of later tiles: on an H100 80GB HBM3 (400 W limit) a cp.async.bulk.prefetch of the next tile made
              // the headline encode 22 % slower and one two tiles ahead another 23 % slower (DESIGN §4 "what binds")
            }
          } else {               // last tiles of the shard: per-row boxes, zero padding via out-of-bounds fill
            if (part == 0) mbar_expect_tx(bar, static_cast<uint32_t>(k) * eb * kRaw3);
            for (int t = part; t < k; t += parts)
              tma_load_2d(dst0 + static_cast<uint32_t>(t) * group_bytes, &maps.m[0], (p.in_c0[t] + i * kTile) >> 2,
                          static_cast<int32_t>(b0), bar);
          }
        } else if (p.tma_mode == kLoadTmaBlocks2D) {
          if (part == 0) mbar_expect_tx(bar, static_cast<uint32_t>(k) * eb * rawp);
          for (int t = part; t < k; t += parts)
            tma_load_2d(dst0 + static_cast<uint32_t>(t) * group_bytes, &maps.m[0], (p.in_c0[t] + i * kTile) >> 2,
                        static_cast<int32_t>(b0), bar);
        } else if (p.tma_mode == kLoadTmaRuns) {
          // survivors that sit at a uniform stride (one staging arena, or shard files of one allocation) arrive with ONE 3-D
          // request per run — (x, erasure block, row) — instead of one 2-D request per row from every warp
          if (part == 0) {
            mbar_expect_tx(bar, static_cast<uint32_t>(k) * eb * rawp);
            for (int q = 0; q < p.nruns; q++)
              tma_load_3d(dst0 + static_cast<uint32_t>(p.run_row0[q]) * group_bytes, &maps.m[q], (p.in_c0[p.run_row0[q]] + i * kTile) >> 2,
                          static_cast<int32_t>(b0), 0, bar);
          }
        } else {  // one map per input stream: rows = erasure blocks of that stream, box {272 B, eb blocks}
          if (part == 0) mbar_expect_tx(bar, static_cast<uint32_t>(k) * eb * rawp);
          for (int t = part; t < k; t += parts)
            tma_load_2d(dst0 + static_cast<uint32_t>(t) * group_bytes, &maps.m[t], (p.in_c0[t] + i * kTile) >> 2,
                        static_cast<int32_t>(b0), bar);
        }
      } else {
        const int per_t = eb * kTile;
        for (int idx = tid; idx < k * per_t; idx += nthr) {
          const int t = idx / per_t, q = idx - t * per_t, e = q >> 8, x = q & (kTile - 1);
          const int64_t xg = static_cast<int64_t>(i) * kTile + x;
          int64_t valid = p.in_limit - static_cast<int64_t>(t) * p.in_shard_step;
          valid = valid < 0 ? 0 : (valid > S ? S : valid);
          uint8_t v = 0;
          if (e < nb && xg < valid) v = p.in_ptr[t][(b0 + e) * p.in_block_stride + xg];
          s_raw[static_cast<uint32_t>(t) * group_bytes + e * rawp + x] = v;
        }
      }
    };
    auto issue_tile = [&](int i) { issue_tile_at(i, b0, nb, 0, 1); };

    if constexpr (USE_TMA) {
      if (warp0) {
        if (elect_one() && ntiles > 0) {
          if constexpr (AUTO) {  // the previous group's last raw tile must have been read by every warp
            if (g != static_cast<int64_t>(blockIdx.x)) mbar_wait(smem_u32(&bars[2]), (it - 1u) & 1u);
          }
          issue_tile(0);
          if constexpr (DIRECT) {
            if (ntiles > 1) issue_tile(1);
          }
        }
        __syncwarp();
      }
    } else {
      if (ntiles > 0) issue_tile(0);
      __syncthreads();
    }

    // ---- HH step: packets [8j, 8j+8) of every stream, from the aligned + output tiles
    // FAST: a full tile of a full group — all eight packets present, no remainder, every hash thread live
    auto hh_step = [&](int j, auto fast_) {
      constexpr bool FAST = decltype(fast_)::value;
      if (FAST ? hh_thread : hh_live) {
        const uint32_t flip = (DIRECT && ((it + static_cast<uint32_t>(j)) & 1u)) ? hh_flip : 0u;
        const uint32_t addr = hh_addr + flip;
        const int q0 = 8 * j;
        if (FAST || q0 + 8 <= npk) {
#pragma unroll
          for (int q = 0; q < 8; q++) {
            const uint4 v = lds128(addr + 32 * q);
            hh_update(hs, pack64(v.x, v.y), pack64(v.z, v.w));
          }
        } else {
#pragma unroll 1
          for (int q = 0; q0 + q < npk; q++) {
            const uint4 v = lds128(addr + 32 * q);
            hh_update(hs, pack64(v.x, v.y), pack64(v.z, v.w));
          }
        }
        if (!FAST && j == ntiles - 1 && rem) {
          const uint8_t* tail = hh_row + flip + ((npk * 32) & (kTile - 1));
          hh_remainder(hs, h, rem, [&](int idx) -> uint32_t { return tail[idx]; });
        }
      }
    };

    // ---------------- one tile.  The steady state (FAST: every byte of the tile inside the shard, every block of the group
    // present) carries no bounds predicates and no partial stores; only the last tile of a shard and the last, partial
    // group of a launch take the general form.
    auto tile_body = [&](int i, auto fast_) {
      constexpr bool FAST = decltype(fast_)::value;
      const uint32_t sel = DIRECT ? ((it + static_cast<uint32_t>(i)) & 1u) : 0u;
      MEC_PHASE_SKIP();
      if constexpr (DIRECT) mbar_wait(smem_u32(&bars[sel]), ((it + static_cast<uint32_t>(i)) >> 1) & 1u);
      else if constexpr (USE_TMA) mbar_wait(smem_u32(&bars[0]), (it + i) & 1u);
      MEC_PHASE(kPhTma);

      // ---- GF step on tile i: re-align, re-store, multiply, store
      for (int c = tid; c < ncol; c += nthr) {
        const int e = c >> 5, x8 = c & 31;
        const uint8_t* rcol = s_raw + sel * buf_bytes + e * rawp + x8 * 8;
        uint8_t* crow = s_clean + static_cast<uint32_t>(e * k) * kRowPitch + x8 * 8;
        uint8_t* prow = s_par + static_cast<uint32_t>(e) * par_blk + x8 * 8;
        const int64_t xg = static_cast<int64_t>(i) * kTile + x8 * 8;
        uint8_t* gout = p.out + (b0 + e) * r * p.out_pitch + xg;
        const bool full = FAST || (e < nb && xg + 8 <= S);
        const bool part = !FAST && e < nb && xg < S && !full;
        auto store_out = [&](int j, uint2 o) {
          *reinterpret_cast<uint2*>(prow + static_cast<uint32_t>(j) * par_row) = o;
          uint8_t* gp = gout + j * p.out_pitch;
          if (FAST || full) {
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
            uint2 v;
            if constexpr (ALIGN == kAlignRuntime) v = load_col_rt(rcol + t * group_bytes, p.in_align[t]);
            else v = load_col_ct<ROWS3D ? row_lead_3d(t, kSm3, kRG) : ((t * ALIGN) & 15)>(rcol + t * group_bytes);
            lo[t] = v.x; hi[t] = v.y;
            if constexpr (!DIRECT) *reinterpret_cast<uint2*>(crow + t * kRowPitch) = v;
          });
          if constexpr (AUTO && USE_TMA) {
            // the raw tile is dead as soon as every lane holds its column in registers: release it now (one arrival per
            // warp on the "consumed" mbarrier), the issuing lane of warp 0 collects the arrivals before the next TMA batch
            __syncwarp();
            if (elect_one()) mbar_arrive(smem_u32(&bars[2]));
          }
          if constexpr (R > 0) {
            uint32_t olo[R], ohi[R];
            GfStaticApply<typename GF::Mat>::run(lo, olo);
            GfStaticApply<typename GF::Mat>::run(hi, ohi);
#pragma unroll
            for (int j = 0; j < R; j++) store_out(j, make_uint2(olo[j], ohi[j]));
          }
        } else {
          constexpr int RC = GF::RC;
          for (int j0 = 0; j0 < (r > 0 ? r : 1); j0 += RC) {
            uint32_t pl[RC][8], ph[RC][8];
#pragma unroll
            for (int j = 0; j < RC; j++)
#pragma unroll
              for (int b = 0; b < 8; b++) { pl[j][b] = 0u; ph[j][b] = 0u; }
#pragma unroll 2
            for (int t = 0; t < k; t++) {
              uint2 v;
              if constexpr (ALIGN == kAlignRuntime) v = load_col_rt(rcol + t * group_bytes, p.in_align[t]);
              else v = *reinterpret_cast<const uint2*>(rcol + t * group_bytes);
              if constexpr (!DIRECT) { if (j0 == 0) *reinterpret_cast<uint2*>(crow + t * kRowPitch) = v; }
              if (r == 0) continue;
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
              if (j0 + j >= r) break;
              uint32_t al = pl[j][7], ah = ph[j][7];
#pragma unroll
              for (int b = 6; b >= 0; b--) {
                al = gf_xtime_add4(al, pl[j][b]);
                ah = gf_xtime_add4(ah, ph[j][b]);
              }
              store_out(j0 + j, make_uint2(al, ah));
            }
          }
        }
      }
      MEC_PHASE(kPhGf);
      if constexpr (DIRECT) {
        if (r > 0) __syncthreads();  // (A) output rows complete
        MEC_PHASE(kPhBarA);
        hh_step(i, fast_);
        MEC_PHASE(kPhHh);
        __syncthreads();             // (B) everyone is done with this buffer (and the output rows): refill it two tiles ahead
        MEC_PHASE(kPhBarB);
        if (i + 2 < ntiles) {
          if constexpr (ROWS3D) {
            if (warp0) {
              if (elect_one()) issue_tile_at(i + 2, b0, nb, 0, 1);
              __syncwarp();
            }
          } else {
            if (elect_one()) issue_tile_at(i + 2, b0, nb, warp_id, nthr >> 5);
            __syncwarp();
          }
        }
        return;
      }
      if constexpr (AUTO && USE_TMA) {
        static_assert(!AUTO || GF::kIsStatic, "the warp-autonomous pipeline is instantiated for compile-time matrices only");
        __syncwarp();  // (A) this warp's aligned + output rows are complete
        if (warp0 && i + 1 < ntiles) {
          if (elect_one()) {
            mbar_wait(smem_u32(&bars[2]), (it + static_cast<uint32_t>(i)) & 1u);  // every warp holds its columns of tile i
            issue_tile_at(i + 1, b0, nb, 0, 1);
          }
          __syncwarp();
        }
        MEC_PHASE(kPhBarA);
      } else {
        __syncthreads();  // (A) aligned + output tiles complete; raw tile fully consumed
        MEC_PHASE(kPhBarA);
        if (i + 1 < ntiles) {  // refill the raw tile while the hash threads work on the aligned one
          if constexpr (USE_TMA && ROWS3D) {
            if (warp0) {  // a single request per tile: no point in making every warp walk the issue code
              if (elect_one()) issue_tile_at(i + 1, b0, nb, 0, 1);
              __syncwarp();
            }
          } else if constexpr (USE_TMA) {
            if (elect_one()) issue_tile_at(i + 1, b0, nb, warp_id, nthr >> 5);
            __syncwarp();
          } else {
            issue_tile(i + 1);  // visible after barrier (B)
          }
        }
      }

      MEC_PHASE_SKIP();
      hh_step(i, fast_);
      MEC_PHASE(kPhHh);
      // (B) aligned + output rows may be overwritten.  With one warp per erasure block the rows a warp writes in GF(i+1) are
      // read by its own hash lanes only, so the hand-off is warp-local; the raw tile is protected by barrier (A) / the mbarrier
      if constexpr ((AUTO && USE_TMA) || WARP_B) __syncwarp();
      else __syncthreads();
      MEC_PHASE(kPhBarB);
    };
    static_assert(kTile == 256, "tile shift");
    const int nfast = (nb == eb) ? (S >> 8) : 0;
#pragma unroll 1
    for (int i = 0; i < nfast; i++) tile_body(i, std::integral_constant<bool, true>{});
#pragma unroll 1
    for (int i = nfast; i < ntiles; i++) tile_body(i, std::integral_constant<bool, false>{});

    // ---------------- finalisation
    {
      uint64_t d0, d1;
      hh_finalize(hs, d0, d1);  // all threads of the warp take part in the shuffles
      if (hh_live) {
        const int64_t b = b0 + e_hh;
        uint64_t* dg = reinterpret_cast<uint64_t*>(p.digests + (b * nstreams + srow) * 32 + 16 * h);
        dg[0] = d0;
        dg[1] = d1;
        if (!is_out && p.corrupt != nullptr && p.expect_ptr[srow] != nullptr) {
          const uint8_t* ex = p.expect_ptr[srow] + b * p.expect_block_stride + 16 * h;
          uint64_t e0 = 0, e1 = 0;
          for (int q = 0; q < 8; q++) {
            e0 |= static_cast<uint64_t>(ex[q]) << (8 * q);
            e1 |= static_cast<uint64_t>(ex[8 + q]) << (8 * q);
          }
          if (e0 != d0 || e1 != d1) p.corrupt[b * k + srow] = 1;
        }
      }
    }
    it += static_cast<uint32_t>(ntiles);
    if (p.work_counter != nullptr) {
      if (tid == 0) *s_next = claimed;
      __syncthreads();
      g = static_cast<int64_t>(gridDim.x) + *s_next;
      __syncthreads();  // nobody may still be reading the slot when the next group's claim lands
    } else {
      g += gridDim.x;
    }
  }
#if MEC_PHASE_CYCLES
  if ((tid & 31) == 0) ph.close64(kPhWarp, clock64v());
  if (tid == 0 && p.phase != nullptr) {
    const uint64_t ns = global_ns();
    ph.close64(kPhCtaClk, clock64v());
    ph.close64(kPhCtaNs, ns);
    atomicMax(p.phase + 1, static_cast<unsigned long long>(ns));
  }
#endif
}

}  // namespace mec
