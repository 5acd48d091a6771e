// ec_engine.h — host-side engine behind the C ABI: kernel dispatch, tensor maps, device staging.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <mutex>
#include <string>
#include <vector>
#include "ec_kernel.cuh"

namespace mec {

void set_last_error(const std::string& s);
const char* get_last_error();

#define MEC_CUDA_OK(expr)                                                                    \
  do {                                                                                       \
    cudaError_t _e = (expr);                                                                 \
    if (_e != cudaSuccess) {                                                                 \
      ::mec::set_last_error(std::string(#expr) + ": " + cudaGetErrorString(_e));             \
      return MEC_ERR_CUDA;                                                                   \
    }                                                                                        \
  } while (0)

// One fused launch over `nblocks` equally shaped erasure blocks (all pointers are device pointers).
struct FusedDesc {
  int k = 0, r = 0;
  const uint8_t* coef = nullptr;   // r x k row-major runtime matrix (ignored when static_encode)
  bool static_encode = false;      // matrix == parity rows of (k, r): compile-time kernels eligible
  int64_t nblocks = 0;
  int32_t S = 0;
  // input addressing
  bool contiguous = true;          // true: Split layout inside contiguous object bytes
  const uint8_t* in_base = nullptr;  // contiguous: first byte of block 0
  int64_t in_block_stride = 0;     // bytes between consecutive blocks (both kinds)
  int64_t in_block_len = 0;        // contiguous: valid object bytes per block (<= k*S)
  const uint8_t* in_ptr[kMaxK] = {};   // !contiguous: shard t, block 0, byte 0
  const uint8_t* map_base[kMaxK] = {}; // !contiguous: 16B-aligned base of the allocation holding input t
  int64_t map_len[kMaxK] = {};         // !contiguous: addressable bytes from map_base[t]
  // outputs
  uint8_t* out = nullptr;
  int64_t out_pitch = 0;
  uint8_t* digests = nullptr;      // nullptr: skip hashing entirely
  bool hash_outputs = true;        // false: only the k inputs are hashed (GET path: reconstructed data needs no digest)
  const uint8_t* expect_ptr[kMaxK] = {};
  int64_t expect_block_stride = 0;
  uint8_t* corrupt = nullptr;
  const uint8_t* key = nullptr;    // 32-byte HighwayHash key (host)
  const int32_t* block_len = nullptr;  // device: per-block shard bytes (<= S); only launches that take the latency kernel (see small_ok)
  const SmallBlock* blocks = nullptr;  // device, contiguous encode: per-block geometry relative to in_base; S = the largest shard length
  // device, latency kernel only: per-block decode plans (r = the largest plan's rows; coef may then be nullptr)
  const SmallPattern* patterns = nullptr;
  const uint16_t* block_pattern = nullptr;  // one entry per block: its plan in `patterns`
  // one block of the launch is an object's short last block (latency kernel only, see small_ok): no table needed
  int64_t tail_block = -1, tail_in_off = -1;  // index; contiguous encode: byte offset from in_base (rows tail_S apart)
  int32_t tail_S = 0, tail_bytes = 0;
};

struct EngineOptions {
  int eb = 0;              // erasure blocks per CTA (0 = auto)
  int force_bytewise = 0;  // 1: never use TMA
  int force_dynamic = 0;   // 1: never use the compile-time specialised GF kernels
  int balance_grid = 0;  // shrink the persistent grid so that every CTA makes the same number of passes
  int grid_mult = 0;       // CTAs per SM (0 = occupancy; the 3-D-fetch encode of misaligned rows is capped at a budget of load bytes in flight)
  int jit = -1;            // decode-matrix kernels specialised at run time with NVRTC: -1 auto (large launches), 0 never, 1 always
  int no_rows3d = 0;       // 1: never use the one-request-per-tile 3-D TMA fetch
  int use_auto = 0;        // 1: warp-autonomous pipeline (no CTA barriers) when k + r == 16; measured slower, off by default
  int64_t chunk_blocks = 0; // host pipeline chunk (0 = auto)
  int64_t small_blocks = -1; // launches of at most this many erasure blocks take the latency kernel (ec_small.cuh); -1: 5 per SM, 0: never
  int static_groups = 1;   // 1 (default): erasure-block groups are dealt to CTAs statically (g += gridDim.x); 0: through a claim counter —
                           // useful when SMs are shared or uneven
};

// Which kernel form a launch_fused call ran (Engine::dispatch_stat, mec_get_stat keys "form_<name>"): the StaticEntry field, the
// runtime-matrix table, the NVRTC specialisation or the latency kernel
enum KernelForm : int {
  kFormSmall = 0, kFormFast3d, kFormFast3dAuto, kFormFast3dSemi, kFormFast, kFormFastAuto, kFormAligned, kFormAlignedAuto,
  kFormRuntime, kFormBytewise, kFormDynAligned, kFormDynRuntime, kFormDynBytewise, kFormJit, kNumForms
};

// What the last launch_fused call that launched a kernel chose (mec_get_stat keys "last_<name>")
struct LaunchRecord {
  int form = -1;
  int eb = 0;            // erasure blocks per CTA (1 for the latency kernel)
  int64_t grid = 0;      // CTAs launched
  int tma_mode = -1;     // LoaderMode; -1 for the latency kernel
  int rows3d = 0, direct = 0;
  int tiles3d = 0;       // FusedParams::tiles_3d (0 without the 3-D fetch)
  int row_chunk = -1;    // index {0, 1, 2} = rows {1, 2, 4} of the runtime-matrix kernel picked; -1 for a compile-time matrix
};

class Engine {
 public:
  explicit Engine(int device);
  ~Engine();
  int init();
  int device() const { return device_; }
  int launch_fused(const FusedDesc& d, const EngineOptions& opt, cudaStream_t st);
  int64_t launches() const { return launches_; }
  void count_launch() { launches_++; }
  int64_t jit_compiles() const;  // process-wide
  int64_t small_limit(const EngineOptions& opt) const { return opt.small_blocks >= 0 ? opt.small_blocks : 5ll * num_sms_; }  // most blocks a latency-kernel launch takes
  bool small_ok(const EngineOptions& opt, int64_t nblocks) const {  // would a launch of nblocks take the latency kernel?
    return nblocks <= small_limit(opt) && opt.eb <= 0 && !opt.force_bytewise && opt.jit != 1 && nblocks < (1ll << 31);
  }
  int64_t small_launches() const { return small_launches_; }  // launches that took the latency kernel (ec_small.cuh)
  int64_t jit_launches() const { return jit_launches_; }  // launches of this engine that ran a specialised kernel
  double jit_seconds() const;
  int64_t jit_disk_hits() const;  // specialised kernels loaded from the on-disk cache instead of compiled (process-wide)
  int num_sms() const { return num_sms_; }
  // dispatch record: launches per kernel form ("form_<name>"), the last launch's shape ("last_<name>") and "num_sms";
  // false for any other name
  bool dispatch_stat(const char* name, int64_t* value) const;
  // queue the specialisation of a reconstruct matrix (r x k rows) on the background compiler, as if the pattern were already warm
  void jit_prewarm(int k, int r, const uint8_t* coef, int eb_t, bool hash_out) {
    jit_kernel(k, r, coef, 0, eb_t, false, hash_out, -1, int64_t{1} << 40);
  }

 private:
  int device_;
  int num_sms_ = 0;
  void* encode_tiled_ = nullptr;  // cuTensorMapEncodeTiled
  int64_t launches_ = 0;
  int64_t jit_launches_ = 0;
  int64_t small_launches_ = 0;
  int64_t form_launches_[kNumForms] = {};
  LaunchRecord last_;
  void record_launch(const LaunchRecord& rec) { form_launches_[rec.form]++; last_ = rec; }
  struct LaunchMemo { const void* fn; int threads; size_t smem; int per_sm; };
  std::vector<LaunchMemo> launch_memo_;
  int raise_smem_limit(const void* kfn, size_t smem);
  uint32_t* claim_slots_ = nullptr;  // ring of per-launch group-claim counters (device)
  uint32_t claim_next_ = 0;
  // run-time specialised kernels, keyed by (k, r, matrix bytes)
  void* jit_kernel(int k, int r, const uint8_t* coef, int align, int eb_t, bool rows3d, bool hash_out, int mode, int64_t in_bytes);
};

// stop background specialisation and wait for a compile in flight (mec_shutdown)
void jit_shutdown();
// NVRTC-compile (not load) the kernel specialised for `coef`; cubin bytes, 0 on a compile error, -1 without libnvrtc
int64_t jit_compile_check(int k, int r, const uint8_t* coef, int align, int eb_t, bool rows3d, bool hash_out);

// Grow-only device / page-locked host buffers, freed by their owner.  ensure(n) keeps the buffer when it already holds n bytes and
// otherwise frees it and allocates n plus slack (device: n/8 + 256, which batch_copy.cuh's tail loads rely on; pinned: n/4 + 4096).
struct DevBuf {
  void* p = nullptr;
  size_t cap = 0;
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  ~DevBuf() { release(); }
  int ensure(size_t n);

 private:
  void release();
};

struct PinBuf {
  void* p = nullptr;
  size_t cap = 0;
  PinBuf() = default;
  PinBuf(const PinBuf&) = delete;
  PinBuf& operator=(const PinBuf&) = delete;
  ~PinBuf() { release(); }
  int ensure(size_t n) {
    if (n <= cap) return MEC_OK;
    release();
    const size_t want = n + (n >> 2) + 4096;
    MEC_CUDA_OK(cudaHostAlloc(&p, want, cudaHostAllocPortable));
    cap = want;
    return MEC_OK;
  }

 private:
  void release() {
    if (p) cudaFreeHost(p);
    p = nullptr;
    cap = 0;
  }
};

// A device table and its page-locked twin: filled on the host and uploaded, or written by a kernel and downloaded for the host to
// read.  Sites that need one side only size that side.
struct Mirror {
  DevBuf d;
  PinBuf h;
  int ensure(size_t n) {
    const int rc = d.ensure(n);
    return rc ? rc : h.ensure(n);
  }
  cudaError_t upload(size_t n, cudaStream_t st) const { return cudaMemcpyAsync(d.p, h.p, n, cudaMemcpyHostToDevice, st); }
  cudaError_t download(size_t n, cudaStream_t st) const { return cudaMemcpyAsync(h.p, d.p, n, cudaMemcpyDeviceToHost, st); }
};

// A CUDA stream / event that stays null until create() and is destroyed by its owner.  create() on one that exists is a no-op.
class Stream {
 public:
  Stream() = default;
  Stream(const Stream&) = delete;
  Stream& operator=(const Stream&) = delete;
  ~Stream() { if (h_) cudaStreamDestroy(h_); }
  cudaError_t create(unsigned flags) { return h_ ? cudaSuccess : cudaStreamCreateWithFlags(&h_, flags); }
  operator cudaStream_t() const { return h_; }

 private:
  cudaStream_t h_ = nullptr;
};

class Event {
 public:
  Event() = default;
  Event(const Event&) = delete;
  Event& operator=(const Event&) = delete;
  ~Event() { if (h_) cudaEventDestroy(h_); }
  cudaError_t create(unsigned flags) { return h_ ? cudaSuccess : cudaEventCreateWithFlags(&h_, flags); }
  operator cudaEvent_t() const { return h_; }

 private:
  cudaEvent_t h_ = nullptr;
};

}  // namespace mec
