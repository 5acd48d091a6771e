// ec_api.cu — the C ABI of include/minio_ec.h on top of the fused kernel engine.
//
// Host-buffer entry points stage through device memory owned by the codec with a kSlots-deep (six-slot)
// H2D -> kernel -> D2H pipeline; *_device entry points run on caller-provided device memory.
// There is NO CPU fallback anywhere in this file: without a usable GPU every call fails.
#include <algorithm>
#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <memory>
#include <thread>
#include <vector>
#include "../../include/minio_ec.h"
#include "ec_engine.h"
#include "whole_hash.cuh"
#include "crc.cuh"
#include "obj_hash.cuh"
#include "batch_copy.cuh"
#include "chacha.cuh"
#include "dare.cuh"
#include "sigv4.cuh"
#include <nvtx3/nvToolsExt.h>

struct NvtxRange {
  explicit NvtxRange(const char* n) { nvtxRangePushA(n); }
  ~NvtxRange() { nvtxRangePop(); }
};

using namespace mec;

static const uint8_t kMagicKey[32] = {  // cmd/bitrot.go:37
    0x4b, 0xe7, 0x34, 0xfa, 0x8e, 0x23, 0x8a, 0xcd, 0x26, 0x3e, 0x83, 0xe6, 0xbb, 0x96, 0x85, 0x52,
    0x04, 0x0f, 0x93, 0x5d, 0xa3, 0x9f, 0x44, 0x14, 0x97, 0xe0, 0x9d, 0x13, 0x22, 0xde, 0x36, 0xa0};

static inline int64_t ceil_frac(int64_t num, int64_t den) {  // cmd/utils.go:689
  if (den == 0) return 0;
  if (den < 0) { num = -num; den = -den; }
  int64_t c = num / den;
  if (num > 0 && num % den != 0) c++;
  return c;
}
static inline int64_t round_up(int64_t v, int64_t a) { return (v + a - 1) / a * a; }

constexpr int kSlots = 6;

struct Slot {
  DevBuf src, out, aux;              // aux: survivor arena of a reconstruct chunk / shard files of the whole-file path
  Mirror dig, flags;                 // digests and digest verdicts: small, read by the host right after the stream drains
  // object checksums of an encode chunk (crc.cuh); of a merged batch: per-item partials (crc_part), per-request results (crc_out)
  DevBuf crc_part;
  Mirror crc_out;
  Mirror crc_tab;                    // checksum work table of a merged batch ([CrcReq nreq][CrcWork nwork], crc.cuh)
  Mirror dreq;                       // request table of a merged batch (batch_copy.cuh)
  Mirror blk;                        // per-block geometry of a merged launch (SmallBlock / per-frame lengths)
  Mirror sum_tab, sum_out;           // object hashes of a merged batch: SumWork table, one kSumRecord record per request (obj_hash.cuh)
  // merged batches with whole-file readers (batch_whole_stage): the WholeStream of every staged shard file (whole_hash.cuh) and
  // each request's first stream behind them; one 64-byte digest per staged file
  Mirror wtab, wdig;
  Mirror dpk;                        // mec_encode_sse: the DarePkg rows of the chunk's packages; a merged batch: of all its packages
  // merged batches with encrypted requests (mec_batcher_encode_sse / _decode_sse): the streams' DareStreamKeys and their host-written
  // heads, the plaintext arena, and the package verdicts of an open
  DevBuf sse_keys, sse_pt;
  PinBuf hsse_keys;
  Mirror sse_st;
  int64_t sse_heads = 0;             // key heads written to hsse_keys by the slot's batch in flight (zeroed by batcher_finish)
  // mec_encode_chunked: the signature rows of the chunk and their verdicts behind them; the second stream that verifies them while
  // s.st encodes, with the events that order it after the staging and s.st after it
  Mirror sig_tab;
  Stream st, st2;
  Event ev_staged, ev_verified;
};

// DARE 2.0 state of a codec (dare.cuh): the AES round tables (built once), the key schedules and H powers of the streams of the
// call in flight (zeroed before the call returns), a package table and its verdicts; mec_decode_sse's ciphertext and plaintext
// of the range.
struct DareState {
  bool tabs_ok = false;
  DevBuf tabs, keys, ct, pt;
  PinBuf hkeys;
  Mirror pk, st;
};

// Signature V4 streaming state of a codec (sigv4.cuh): the SigCall of the call in flight (key states zeroed before it returns) and
// mec_chunk_signatures_device's row table with the verdicts behind the rows.
struct SigState {
  Mirror call, rows;
};

struct mec_codec {
  int k = 0, m = 0, n = 0;
  int64_t block_size = 0;
  int algo = 0, device = 0;
  std::vector<uint8_t> matrix;  // n x k
  std::unique_ptr<Engine> eng;
  EngineOptions opt;
  std::mutex mu;
  Slot slots[kSlots];
  DevBuf flags, crc_tables;
  std::unique_ptr<CrcTables> crc_host;  // host copy of the CRC tables (combine across chunks)
  int checksums = 0;                    // option "checksums": MEC_CRC32 | MEC_CRC32C | MEC_CRC64NVME computed by the host-buffer encode calls
  uint64_t last_crc[kCrcTypes] = {0, 0, 0};
  int64_t last_crc_len = 0;
  // mec_sums_device: the work table of the last call, and an event behind its kernel (the next call refills the table after it)
  Mirror sum_tab;
  Event sum_ev;
  // boundary counters (mec_get_stat)
  int64_t st_blocks_encoded = 0, st_blocks_read = 0, st_shards_rebuilt = 0, st_corrupt = 0, st_h2d = 0, st_d2h = 0;
  int64_t st_whole_hash = 0;  // whole_hash_kernel launches
  // mec_decode_mixed / mec_heal_mixed: the verified whole-file readers of the call (k files at a pitch of round_up(sfs, 16) + 256)
  // and their digests; they stay on the device for the whole call while the slot arenas cycle through the chunks
  DevBuf whole;
  Mirror whole_dig;
  DareState dare;
  int64_t st_dare_sealed = 0, st_dare_opened = 0;  // DARE packages sealed / opened (rows launched, each once whatever its cipher)
  std::atomic<int> dare_chacha20{0};  // option "dare_chacha20": 0 AES-256-GCM only; 1 also open ChaCha20-Poly1305; 2 also seal with it
  SigState sig;
  int64_t st_sigv4_chunks = 0;  // signature rows verified
  int64_t S() const { return ceil_frac(block_size, k); }
};

// Drains slot streams on every return, errors included, so that no copy a failed call enqueued is still writing into caller
// memory (or reading staging the next call reuses) when the caller sees the error code.  Every slot, or the one slot of a
// whole-file path.
struct SlotDrain {
  Slot* s;
  int n;
  explicit SlotDrain(mec_codec* c) : s(c->slots), n(kSlots) {}
  explicit SlotDrain(Slot& one) : s(&one), n(1) {}
  ~SlotDrain() { for (int i = 0; i < n; i++) if (s[i].st) cudaStreamSynchronize(s[i].st); }
};

// The codec's slots as a round-robin ring for pipelines that retire their chunks in submission order.  acquire() syncs slot `si`
// and retires the chunk it carried; submitted() marks it busy and moves on; finish() retires everything still in flight, oldest
// first.  retire(si) runs on the host once slot si's stream has drained.
template <class Retire>
struct SlotRing {
  mec_codec* c;
  Retire retire;
  bool busy[kSlots] = {};
  int si = 0;
  SlotRing(mec_codec* c_, Retire r) : c(c_), retire(r) {}
  int acquire() {
    MEC_CUDA_OK(cudaStreamSynchronize(c->slots[si].st));
    if (busy[si]) { retire(si); busy[si] = false; }
    return MEC_OK;
  }
  void submitted() { busy[si] = true; si = (si + 1) % kSlots; }
  int finish() {
    for (int q = 0; q < kSlots; q++, si = (si + 1) % kSlots) {
      MEC_CUDA_OK(cudaStreamSynchronize(c->slots[si].st));
      if (busy[si]) { retire(si); busy[si] = false; }
    }
    return MEC_OK;
  }
};

// ------------------------------------------------------------------------------------------------
extern "C" int mec_device_count(void) {
  int c = 0;
  if (cudaGetDeviceCount(&c) != cudaSuccess) return 0;
  return c;
}
extern "C" const char* mec_last_error(void) { return get_last_error(); }
extern "C" const char* mec_version(void) { return "minio_b200 0.1 (sm_90a; fused RS+HighwayHash256)"; }

extern "C" int64_t mec_ceil_frac(int64_t a, int64_t b) { return ceil_frac(a, b); }
extern "C" int64_t mec_shard_size(const mec_codec* c) { return c->S(); }
extern "C" int64_t mec_shard_file_size(const mec_codec* c, int64_t total) {
  if (total == 0) return 0;
  if (total == -1) return -1;
  const int64_t num = total / c->block_size, last = total % c->block_size;
  return num * c->S() + ceil_frac(last, c->k);
}
extern "C" int64_t mec_shard_file_offset(const mec_codec* c, int64_t start, int64_t length, int64_t total) {
  const int64_t ss = c->S(), sfs = mec_shard_file_size(c, total);
  const int64_t end_shard = (start + length) / c->block_size;
  return std::min(end_shard * ss + ss, sfs);
}
extern "C" int64_t mec_bitrot_shard_file_size(int64_t size, int64_t shard_size, int algo) {
  if (algo != MEC_HIGHWAYHASH256S) return size;
  return ceil_frac(size, shard_size) * 32 + size;
}

extern "C" int mec_codec_new(int k, int m, int64_t block_size, int algo, int device, mec_codec** out) {
  if (!out) return MEC_ERR_INVALID_ARGUMENT;
  *out = nullptr;
  if (k <= 0 || m < 0) return MEC_ERR_INV_SHARD_NUM;   // cmd/erasure-coding.go:44-46
  if (k + m > 256) return MEC_ERR_MAX_SHARD_NUM;       // cmd/erasure-coding.go:48-50
  if (block_size <= 0) return MEC_ERR_INVALID_ARGUMENT;
  if (algo < MEC_SHA256 || algo > MEC_BLAKE2B512) return MEC_ERR_INVALID_ARGUMENT;
  std::unique_ptr<mec_codec> c(new mec_codec);
  c->k = k; c->m = m; c->n = k + m; c->block_size = block_size; c->algo = algo; c->device = device;
  c->matrix.resize(static_cast<size_t>(c->n) * k);
  if (!rs_coding_matrix(k, m, c->matrix.data())) return MEC_ERR_INV_SHARD_NUM;
  if (const char* e = getenv("MEC_EB")) c->opt.eb = atoi(e);
  if (const char* e = getenv("MEC_FORCE_BYTEWISE")) c->opt.force_bytewise = atoi(e);
  if (const char* e = getenv("MEC_FORCE_DYNAMIC")) c->opt.force_dynamic = atoi(e);
  if (const char* e = getenv("MEC_GRID_MULT")) c->opt.grid_mult = atoi(e);
  if (const char* e = getenv("MEC_BALANCE_GRID")) c->opt.balance_grid = atoi(e);
  if (const char* e = getenv("MEC_CHUNK_BLOCKS")) c->opt.chunk_blocks = atoll(e);
  if (const char* e = getenv("MEC_USE_AUTO")) c->opt.use_auto = atoi(e);
  if (const char* e = getenv("MEC_JIT")) c->opt.jit = atoi(e);
  if (const char* e = getenv("MEC_NO_ROWS3D")) c->opt.no_rows3d = atoi(e);
  if (const char* e = getenv("MEC_SMALL_BLOCKS")) c->opt.small_blocks = atoll(e);
  if (const char* e = getenv("MEC_STATIC_GROUPS")) c->opt.static_groups = atoi(e);
  *out = c.release();
  return MEC_OK;
}

// The encoder is created on first use (like the sync.Once in cmd/erasure-coding.go:59-71); without a
// usable GPU this fails loudly — there is no CPU path behind this ABI.
static int ensure_engine(mec_codec* c) {
  if (c->eng) return MEC_OK;
  std::unique_ptr<Engine> e(new Engine(c->device));
  int rc = e->init();
  if (rc) return rc;
  for (auto& s : c->slots)
    if (s.st.create(cudaStreamNonBlocking) != cudaSuccess) {
      set_last_error(std::string("cudaStreamCreate: ") + cudaGetErrorString(cudaGetLastError()));
      return MEC_ERR_CUDA;
    }
  c->eng = std::move(e);
  return MEC_OK;
}

extern "C" void mec_codec_free(mec_codec* c) {
  if (!c) return;
  if (c->eng) {
    // every slot's streams drain before any stream, event or buffer of the codec is destroyed
    cudaSetDevice(c->device);
    for (auto& s : c->slots) {
      if (s.st) cudaStreamSynchronize(s.st);
      if (s.st2) cudaStreamSynchronize(s.st2);
    }
  }
  delete c;
}

extern "C" int mec_set_option(mec_codec* c, const char* name, int64_t v) {
  if (!c || !name) return MEC_ERR_INVALID_ARGUMENT;
  std::lock_guard<std::mutex> lk(c->mu);
  if (!strcmp(name, "eb")) c->opt.eb = static_cast<int>(v);
  else if (!strcmp(name, "force_bytewise")) c->opt.force_bytewise = static_cast<int>(v);
  else if (!strcmp(name, "force_dynamic")) c->opt.force_dynamic = static_cast<int>(v);
  else if (!strcmp(name, "grid_mult")) c->opt.grid_mult = static_cast<int>(v);
  else if (!strcmp(name, "balance_grid")) c->opt.balance_grid = static_cast<int>(v);
  else if (!strcmp(name, "use_auto")) c->opt.use_auto = static_cast<int>(v);
  else if (!strcmp(name, "jit")) c->opt.jit = static_cast<int>(v);
  else if (!strcmp(name, "no_rows3d")) c->opt.no_rows3d = static_cast<int>(v);
  else if (!strcmp(name, "chunk_blocks")) c->opt.chunk_blocks = v;
  else if (!strcmp(name, "static_groups")) c->opt.static_groups = static_cast<int>(v);
  else if (!strcmp(name, "small_blocks")) c->opt.small_blocks = v;
  else if (!strcmp(name, "checksums")) c->checksums = static_cast<int>(v) & 7;
  else if (!strcmp(name, "dare_chacha20")) {
    if (v < 0 || v > 2) return MEC_ERR_INVALID_ARGUMENT;
    c->dare_chacha20 = static_cast<int>(v);
  }
  else return MEC_ERR_INVALID_ARGUMENT;
  return MEC_OK;
}
// non-zero bytes of signing-key material left in the codec: the host copy of the key states and a read-back of the device copy
static int64_t sig_key_bytes(const mec_codec* c) {
  const size_t kb = offsetof(SigCall, head_len);
  int64_t nz = 0;
  for (int dev = 0; dev < 2; dev++) {
    const void* p = dev ? c->sig.call.d.p : c->sig.call.h.p;
    if (!p) continue;
    uint8_t buf[offsetof(SigCall, head_len)];
    if (dev) {
      if (cudaSetDevice(c->device) != cudaSuccess || cudaMemcpy(buf, p, kb, cudaMemcpyDeviceToHost) != cudaSuccess) return -1;
    } else {
      memcpy(buf, p, kb);
    }
    for (size_t i = 0; i < kb; i++) nz += buf[i] != 0;
  }
  return nz;
}

extern "C" int64_t mec_get_stat(const mec_codec* c, const char* name) {
  if (!c || !name) return -1;
  if (!strcmp(name, "launches")) return c->eng ? c->eng->launches() : 0;
  if (!strcmp(name, "blocks_encoded")) return c->st_blocks_encoded;
  if (!strcmp(name, "blocks_read")) return c->st_blocks_read;
  if (!strcmp(name, "shards_rebuilt")) return c->st_shards_rebuilt;
  if (!strcmp(name, "corrupt_shards")) return c->st_corrupt;
  if (!strcmp(name, "bytes_h2d")) return c->st_h2d;
  if (!strcmp(name, "bytes_d2h")) return c->st_d2h;
  if (!strcmp(name, "whole_hash_launches")) return c->st_whole_hash;
  if (!strcmp(name, "dare_sealed")) return c->st_dare_sealed;
  if (!strcmp(name, "dare_opened")) return c->st_dare_opened;
  if (!strcmp(name, "dare_chacha20")) return c->dare_chacha20.load();
  if (!strcmp(name, "sigv4_chunks")) return c->st_sigv4_chunks;
  if (!strcmp(name, "sigv4_key_bytes")) return sig_key_bytes(c);
  if (!strcmp(name, "jit_compiles")) return c->eng ? c->eng->jit_compiles() : 0;
  if (!strcmp(name, "jit_launches")) return c->eng ? c->eng->jit_launches() : 0;
  if (!strcmp(name, "small_launches")) return c->eng ? c->eng->small_launches() : 0;
  if (!strcmp(name, "jit_ms")) return c->eng ? static_cast<int64_t>(c->eng->jit_seconds() * 1e3) : 0;
  if (!strcmp(name, "jit_disk_hits")) return c->eng ? c->eng->jit_disk_hits() : 0;
  static const Engine kNoLaunches(0);  // dispatch record of a handle that has not launched yet
  int64_t v = 0;
  if ((c->eng ? *c->eng : kNoLaunches).dispatch_stat(name, &v)) return v;
  return -1;
}
extern "C" void mec_shutdown(void) { mec::jit_shutdown(); }

extern "C" int64_t mec_jit_compile_check(int k, int r, const uint8_t* coef, int align, int eb, int rows3d, int hash_outputs) {
  if (k < 1 || k > kMaxK || r < 1 || r > kMaxR || !coef || align < 0 || align > 15 || eb < 0) return MEC_ERR_INVALID_ARGUMENT;
  return mec::jit_compile_check(k, r, coef, align, eb, rows3d != 0, hash_outputs != 0);
}

// What a read through k readers rebuilds, and how (parallelReader.Read + reedsolomon's Reconstruct, cmd/erasure-decode.go:145-221):
// every wanted shard that is not read is a target; rows are the r x k decode rows that rebuild the targets from the read shards.
struct DecodePlan {
  uint8_t present[kMaxShards] = {};  // shard i is one of the k readers
  int targets[kMaxShards];
  int r = 0;
  std::vector<uint8_t> rows;  // r x k (one zero row when r == 0)
};

// chosen[0..nch): the readers in ascending shard order, of which the first k are read.  want == NULL wants every shard;
// data_only leaves the parity shards out.
static int plan_decode(const mec_codec* c, const int* chosen, int nch, const uint8_t* want, int data_only, DecodePlan* p) {
  const int k = c->k;
  if (nch < k) return MEC_ERR_READ_QUORUM;
  memset(p->present, 0, sizeof(p->present));
  for (int t = 0; t < k; t++) p->present[chosen[t]] = 1;
  p->r = 0;
  for (int i = 0; i < c->n; i++)
    if ((!want || want[i]) && !p->present[i] && !(data_only && i >= k)) p->targets[p->r++] = i;
  if (p->r > kMaxR) return MEC_ERR_UNSUPPORTED;
  p->rows.assign(static_cast<size_t>(std::max(p->r, 1)) * k, 0);
  int valid[kMaxShards];
  if (p->r > 0 && !rs_decode_rows(k, c->m, p->present, p->targets, p->r, p->rows.data(), valid)) return MEC_ERR_TOO_FEW_SHARDS;
  return MEC_OK;
}

// Pre-warm the kernel cache for the erasure patterns a drive failure will produce: every single missing data shard (the degraded
// GET of cmd/erasure-decode.go:239 with one drive gone, and the heal of that drive), both CTA shapes.  Compiles run on the
// background thread (and land in the on-disk cache), nothing waits for them.
extern "C" int mec_jit_prewarm(mec_codec* c) {
  if (!c) return MEC_ERR_INVALID_ARGUMENT;
  std::lock_guard<std::mutex> lk(c->mu);
  int rc = ensure_engine(c);
  if (rc) return rc;
  const int k = c->k, n = c->n;
  if (k > kMaxK || n > kMaxShards || c->m < 1) return 0;
  int queued = 0;
  for (int miss = 0; miss < k; miss++) {
    int chosen[kMaxK], cnt = 0;
    uint8_t want[kMaxShards] = {};
    want[miss] = 1;
    for (int i = 0; i < n && cnt < k; i++)
      if (i != miss) chosen[cnt++] = i;
    DecodePlan p;
    if (plan_decode(c, chosen, cnt, want, 0, &p)) continue;
    for (int eb_t : {4, 0})
      for (bool hash_out : {false, true}) {
        c->eng->jit_prewarm(k, 1, p.rows.data(), eb_t, hash_out);
        queued++;
      }
  }
  return queued;
}

extern "C" int64_t mec_launch_count(const mec_codec* c) { return (c && c->eng) ? c->eng->launches() : 0; }

static int require_streaming(mec_codec* c) {
  if (c->algo != MEC_HIGHWAYHASH256S) {
    set_last_error("only HighwayHash256S (streaming bitrot) is implemented on the GPU path");
    return MEC_ERR_UNSUPPORTED;
  }
  std::lock_guard<std::mutex> lk(c->mu);
  return ensure_engine(c);
}

// ------------------------------------------------------------------------------------------------
// object checksums (internal/hash/checksum.go, crc.go): CRC32 / CRC32C / CRC64NVME of a byte stream that is already in HBM
static int ensure_crc(mec_codec* c) {
  if (c->crc_host) return MEC_OK;
  std::unique_ptr<CrcTables> t(new CrcTables);
  crc_build_tables(t.get());
  int rc = c->crc_tables.ensure(sizeof(CrcTables));
  if (rc) return rc;
  MEC_CUDA_OK(cudaMemcpy(c->crc_tables.p, t.get(), sizeof(CrcTables), cudaMemcpyHostToDevice));
  c->crc_host = std::move(t);
  return MEC_OK;
}
// enqueue: CRCs of d_src[0, len) -> d_out3 (device, kCrcTypes words); `part` is scratch for the per-region partials
static int checksums_enqueue(mec_codec* c, const uint8_t* d_src, int64_t len, int which, DevBuf& part, uint64_t* d_out3, cudaStream_t st) {
  int rc = ensure_crc(c);
  if (rc) return rc;
  CrcParams p;
  p.src = d_src; p.len = len; p.which = which & 7;
  p.tables = static_cast<const CrcTables*>(c->crc_tables.p);
  p.nregions = (len + kCrcRegion - 1) / kCrcRegion;
  if ((rc = part.ensure(static_cast<size_t>(std::max<int64_t>(p.nregions, 1)) * kCrcTypes * sizeof(uint64_t)))) return rc;
  p.partial = static_cast<uint64_t*>(part.p);
  p.out = d_out3;
  if (p.nregions > 0) {
    const unsigned grid = static_cast<unsigned>(std::min<int64_t>(p.nregions, static_cast<int64_t>(c->eng->num_sms()) * 8));
    crc_regions_kernel<<<grid, kCrcThreads, 0, st>>>(p);
    MEC_CUDA_OK(cudaGetLastError());
    c->eng->count_launch();
  }
  crc_fold_kernel<<<1, kCrcThreads, 0, st>>>(p);
  MEC_CUDA_OK(cudaGetLastError());
  c->eng->count_launch();
  return MEC_OK;
}

extern "C" uint64_t mec_checksum_combine(int type, uint64_t crc1, uint64_t crc2, int64_t len2) {
  const int ty = type == MEC_CRC32 ? 0 : (type == MEC_CRC32C ? 1 : (type == MEC_CRC64NVME ? 2 : -1));
  if (ty < 0) return 0;
  static const CrcTables* tabs = [] { CrcTables* t = new CrcTables; crc_build_tables(t); return t; }();
  const CrcSpec sp = crc_spec(ty);
  return crc_combine(tabs->xp8[ty], crc1, crc2, len2, sp.poly, sp.bits);  // Checksum.AddPart (internal/hash/crc.go:32-73)
}

extern "C" int mec_checksums_device(mec_codec* c, const uint8_t* d_src, int64_t len, int which, uint64_t* out3, void* stream) {
  if (!c || len < 0 || !out3 || (len > 0 && !d_src)) return MEC_ERR_INVALID_ARGUMENT;
  std::lock_guard<std::mutex> lk(c->mu);
  int rc = ensure_engine(c);
  if (rc) return rc;
  MEC_CUDA_OK(cudaSetDevice(c->device));
  Slot& s = c->slots[0];
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if ((rc = s.crc_out.d.ensure(kCrcTypes * sizeof(uint64_t)))) return rc;
  if ((rc = checksums_enqueue(c, d_src, len, which, s.crc_part, static_cast<uint64_t*>(s.crc_out.d.p), st))) return rc;
  MEC_CUDA_OK(cudaMemcpyAsync(out3, s.crc_out.d.p, kCrcTypes * sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
  MEC_CUDA_OK(cudaStreamSynchronize(st));
  return MEC_OK;
}

// ------------------------------------------------------------------------------------------------
// object hashes (obj_hash.cuh): MD5 / SHA-1 / SHA-256 of many two-segment messages in device memory, one thread per (message,
// algorithm).  The host writes the work table, sorted by (algorithm, length descending) so that a warp runs one algorithm over
// similar lengths; mec_sums_device and the coalescer's PUT batches share this table code and the launch.
constexpr int kSumMask = MEC_SUM_MD5 | MEC_SUM_SHA1 | MEC_SUM_SHA256;
static_assert(MEC_SUM_BYTES == kSumRecord && MEC_SUM_MD5 << 1 == MEC_SUM_SHA1 && MEC_SUM_MD5 << 2 == MEC_SUM_SHA256, "obj_hash.cuh");

// appends the items of one message (segments at off0 / off1 of the base buffer) whose record is at byte `rec` of the output
static int64_t sum_items(SumWork* t, int64_t w, int which, int64_t rec, int64_t off0, int64_t len0, int64_t off1, int64_t len1) {
  for (int a = 0; a < kSumAlgos; a++)
    if (which & (MEC_SUM_MD5 << a)) t[w++] = SumWork{off0, len0, off1, len1, rec + 32 * a, a, 0};
  return w;
}
static void sum_sort(SumWork* t, int64_t n) {
  std::sort(t, t + n, [](const SumWork& x, const SumWork& y) {
    return x.algo != y.algo ? x.algo < y.algo : x.len0 + x.len1 > y.len0 + y.len1;
  });
}
// enqueue: ONE stream_sums_kernel over the nwork items of the device table `work`
static int sum_launch(mec_codec* c, const uint8_t* base, const SumWork* work, int64_t nwork, uint8_t* out, cudaStream_t st) {
  SumParams p;
  p.base = base; p.work = work; p.nwork = nwork; p.out = out;
  stream_sums_kernel<<<static_cast<unsigned>(ceil_frac(nwork, kSumThreads)), kSumThreads, 0, st>>>(p);
  MEC_CUDA_OK(cudaGetLastError());
  c->eng->count_launch();
  return MEC_OK;
}

extern "C" int mec_sums_device(mec_codec* c, int which, const uint8_t* d_base, const int64_t* offsets, const int64_t* lens,
                               int64_t count, uint8_t* d_sums, void* stream) {
  if (!c || which <= 0 || (which & ~kSumMask) || count < 0) return MEC_ERR_INVALID_ARGUMENT;
  if (count == 0) return MEC_OK;
  if (!offsets || !lens || !d_sums) return MEC_ERR_INVALID_ARGUMENT;
  for (int64_t i = 0; i < count; i++)
    if (offsets[i] < 0 || lens[i] < 0 || (lens[i] > 0 && !d_base)) return MEC_ERR_INVALID_ARGUMENT;
  const int per = __builtin_popcount(static_cast<unsigned>(which));
  if (count > (int64_t{1} << 36) / per) return MEC_ERR_UNSUPPORTED;  // the grid's x dimension
  std::lock_guard<std::mutex> lk(c->mu);
  int rc;
  if ((rc = ensure_engine(c))) return rc;
  MEC_CUDA_OK(cudaSetDevice(c->device));
  MEC_CUDA_OK(c->sum_ev.create(cudaEventDisableTiming));
  MEC_CUDA_OK(cudaEventSynchronize(c->sum_ev));  // the previous call's kernel has read its table
  const int64_t nwork = count * per;
  const size_t bytes = static_cast<size_t>(nwork) * sizeof(SumWork);
  if ((rc = c->sum_tab.ensure(bytes))) return rc;
  SumWork* t = static_cast<SumWork*>(c->sum_tab.h.p);
  int64_t w = 0;
  for (int64_t i = 0; i < count; i++) w = sum_items(t, w, which, i * kSumRecord, offsets[i], lens[i], 0, 0);
  sum_sort(t, nwork);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  MEC_CUDA_OK(c->sum_tab.upload(bytes, st));
  if ((rc = sum_launch(c, d_base, static_cast<const SumWork*>(c->sum_tab.d.p), nwork, d_sums, st))) return rc;
  MEC_CUDA_OK(cudaEventRecord(c->sum_ev, st));
  return MEC_OK;
}

extern "C" int mec_checksums(mec_codec* c, const uint8_t* src, int64_t len, int which, uint64_t* out3) {
  if (!c || len < 0 || !out3 || (len > 0 && !src)) return MEC_ERR_INVALID_ARGUMENT;
  std::lock_guard<std::mutex> lk(c->mu);
  int rc = ensure_engine(c);
  if (rc) return rc;
  if ((rc = ensure_crc(c))) return rc;
  MEC_CUDA_OK(cudaSetDevice(c->device));
  SlotDrain drain(c);
  const int64_t chunk = 64ll << 20;
  uint64_t acc[kCrcTypes] = {0, 0, 0};
  int64_t done = 0;
  int64_t clen[kSlots] = {};
  SlotRing ring(c, [&](int si) {
    const uint64_t* h = static_cast<const uint64_t*>(c->slots[si].crc_out.h.p);
    for (int ty = 0; ty < kCrcTypes; ty++) {
      const CrcSpec sp = crc_spec(ty);
      acc[ty] = done == 0 ? h[ty] : crc_combine(c->crc_host->xp8[ty], acc[ty], h[ty], clen[si], sp.poly, sp.bits);
    }
    done += clen[si];
  });
  for (int64_t off = 0; off < len; off += chunk) {
    if ((rc = ring.acquire())) return rc;
    const int si = ring.si;
    Slot& s = c->slots[si];
    const int64_t n = std::min(chunk, len - off);
    if ((rc = s.src.ensure(static_cast<size_t>(round_up(n, 16) + 256)))) return rc;
    if ((rc = s.crc_out.ensure(kCrcTypes * sizeof(uint64_t)))) return rc;
    MEC_CUDA_OK(cudaMemcpyAsync(s.src.p, src + off, static_cast<size_t>(n), cudaMemcpyHostToDevice, s.st));
    if ((rc = checksums_enqueue(c, static_cast<const uint8_t*>(s.src.p), n, which, s.crc_part, static_cast<uint64_t*>(s.crc_out.d.p), s.st))) return rc;
    MEC_CUDA_OK(s.crc_out.download(kCrcTypes * sizeof(uint64_t), s.st));
    clen[si] = n;
    c->st_h2d += n;
    ring.submitted();
  }
  if ((rc = ring.finish())) return rc;
  for (int ty = 0; ty < kCrcTypes; ty++) out3[ty] = (which & (1 << ty)) ? acc[ty] : 0;
  return MEC_OK;
}

extern "C" int64_t mec_last_checksums(const mec_codec* c, uint64_t* out3) {
  if (!c || !out3) return MEC_ERR_INVALID_ARGUMENT;
  for (int ty = 0; ty < kCrcTypes; ty++) out3[ty] = c->last_crc[ty];
  return c->last_crc_len;
}

// An empty object never reaches encode_pipeline, which resets the carried checksums for every other object: its checksums are
// those of the empty stream, (0, 0, 0) over 0 bytes, not what the previous object left behind.
static void reset_last_checksums(mec_codec* c) {
  std::lock_guard<std::mutex> lk(c->mu);
  if (!c->checksums) return;
  for (auto& v : c->last_crc) v = 0;
  c->last_crc_len = 0;
}

// ------------------------------------------------------------------------------------------------
// encode
static int encode_device_locked(mec_codec* c, const uint8_t* d_src, int64_t len, uint8_t* d_parity, int64_t pitch,
                                uint8_t* d_digests, cudaStream_t st) {
  const int64_t bs = c->block_size, S = c->S();
  const int64_t nfull = len / bs, tail = len % bs;
  FusedDesc d;
  d.k = c->k; d.r = c->m;
  d.coef = c->matrix.data() + static_cast<size_t>(c->k) * c->k;
  d.static_encode = true;
  d.contiguous = true;
  d.key = kMagicKey;
  d.out_pitch = pitch;
  if (nfull > 0 && tail > 0 && c->eng->small_ok(c->opt, nfull + 1)) {
    // a small object with a short last block: ONE launch of the latency kernel, the last block carries its own geometry
    d.nblocks = nfull + 1; d.S = static_cast<int32_t>(S);
    d.in_base = d_src; d.in_block_stride = bs; d.in_block_len = bs;
    d.out = d_parity; d.digests = d_digests;
    d.tail_block = nfull; d.tail_in_off = nfull * bs; d.tail_S = static_cast<int32_t>(ceil_frac(tail, c->k)); d.tail_bytes = static_cast<int32_t>(tail);
    return c->eng->launch_fused(d, c->opt, st);
  }
  if (nfull > 0) {
    d.nblocks = nfull; d.S = static_cast<int32_t>(S);
    d.in_base = d_src; d.in_block_stride = bs; d.in_block_len = bs;
    d.out = d_parity; d.digests = d_digests;
    int rc = c->eng->launch_fused(d, c->opt, st);
    if (rc) return rc;
  }
  if (tail > 0) {
    const int64_t St = ceil_frac(tail, c->k);
    d.nblocks = 1; d.S = static_cast<int32_t>(St);
    d.in_base = d_src + nfull * bs; d.in_block_stride = round_up(tail, 16); d.in_block_len = tail;
    d.out = d_parity + nfull * c->m * pitch;
    d.digests = d_digests ? d_digests + nfull * c->n * 32 : nullptr;  // NULL = parity only, for the tail block too
    int rc = c->eng->launch_fused(d, c->opt, st);
    if (rc) return rc;
  }
  return MEC_OK;
}

extern "C" int mec_encode_blocks_device(mec_codec* c, const uint8_t* d_src, int64_t len, uint8_t* d_parity,
                                        int64_t parity_pitch, uint8_t* d_digests, void* stream) {
  NvtxRange nvtx("mec_encode_blocks_device");
  if (!c || len < 0) return MEC_ERR_INVALID_ARGUMENT;
  int rc;
  if (d_digests == nullptr) {  // parity only (whole-file bitrot algorithms hash separately, mec_whole_hash_device)
    std::lock_guard<std::mutex> lk0(c->mu);
    if ((rc = ensure_engine(c))) return rc;
  } else if ((rc = require_streaming(c))) {
    return rc;
  }
  if (len == 0) return MEC_OK;
  if (c->S() >= (1ll << 31)) return MEC_ERR_UNSUPPORTED;
  std::lock_guard<std::mutex> lk(c->mu);
  return encode_device_locked(c, d_src, len, d_parity, parity_pitch, d_digests, static_cast<cudaStream_t>(stream));
}

static int64_t pick_chunk_blocks(const mec_codec* c) {
  if (c->opt.chunk_blocks > 0) return c->opt.chunk_blocks;
  int64_t cb = (64ll << 20) / c->block_size;
  return cb < 1 ? 1 : cb;
}

// One chunk of the host-buffer encode pipeline, as the sinks below see it.
struct EncChunk {
  int64_t b0, nb;      // erasure blocks [b0, b0 + nb) of the call
  int64_t nfull;       // of which full (block_size) blocks; the call's short tail block, if in this chunk, follows them
  int64_t tail;        // bytes of that tail block (0 = none)
  Slot* s;             // slot whose stream carries the chunk
  int64_t pitch;       // parity row pitch
  // where the chunk lives: full blocks contiguous from d_src / d_out ((b*m + j)*pitch) / digests ([b][n][32]); the tail block
  // has its own addresses (right behind the full blocks in the single-caller pipeline, elsewhere in a merged batch)
  const uint8_t* d_src = nullptr; const uint8_t* d_src_tail = nullptr;
  uint8_t* d_out = nullptr;       uint8_t* d_out_tail = nullptr;
  const uint8_t* h_dig = nullptr; const uint8_t* h_dig_tail = nullptr;  // pinned host copies of the digests (frame sinks)
  cudaStream_t st = nullptr;
};

// What a chunk's staging step leaves on the device: the chunk's object bytes (16-byte aligned) and the bytes the option
// "checksums" covers for it.
struct Staged {
  const uint8_t* obj = nullptr;
  const uint8_t* ck = nullptr;
  int64_t ck_len = 0;
};
// the plain staging step: the chunk's object bytes [off, off + bytes) of `src` copied into the slot
static auto plain_stage(mec_codec* c, const uint8_t* src) {
  return [c, src](Slot& s, int64_t off, int64_t bytes, Staged* o) -> int {
    int rc;
    if ((rc = s.src.ensure(static_cast<size_t>(round_up(bytes, 16) + 256)))) return rc;
    MEC_CUDA_OK(cudaMemcpyAsync(s.src.p, src + off, static_cast<size_t>(bytes), cudaMemcpyHostToDevice, s.st));
    c->st_h2d += bytes;
    o->obj = o->ck = static_cast<const uint8_t*>(s.src.p);
    o->ck_len = bytes;
    return MEC_OK;
  };
}

// The six-slot H2D -> fused kernel -> D2H pipeline behind every host-buffer encode entry point, over `len` object bytes.
// `stage(s, off, bytes, &staged)` puts the chunk's object bytes [off, off + bytes) on the device on s.st; `enqueue(ch)` adds the
// chunk's device->host copies to ch.s->st right behind the kernel; `retire(ch)` runs on the host once that stream has
// drained (digest scatter into frames).  On any error every slot stream is drained before returning (SlotDrain).
template <class Stage, class Enqueue, class Retire>
static int encode_pipeline(mec_codec* c, int64_t len, Stage&& stage, Enqueue&& enqueue, Retire&& retire) {
  const int64_t bs = c->block_size, S = c->S(), pitch = round_up(S, 16);
  const int64_t nall = ceil_frac(len, bs);
  int64_t chunk = pick_chunk_blocks(c);
  // an object of a few chunks' worth or less is cut into ~four pieces so that its staging, kernel and copy-back overlap (a launch of
  // a handful of blocks costs the same ~0.16 ms as one of a hundred: for 8-64 MiB objects the copies are what is worth overlapping)
  if (c->opt.chunk_blocks <= 0 && nall < 2 * chunk) chunk = std::max<int64_t>(4, ceil_frac(nall, 4));
  SlotDrain drain(c);
  EncChunk inflight[kSlots];
  int rc;
  // option "checksums": CRCs of the object bytes ride along — computed on the chunk that was just staged for the encode (the
  // bytes cross PCIe once), merged across chunks on the host the way Checksum.AddPart merges parts
  const int ck = c->checksums;
  int64_t ck_len[kSlots] = {}, ck_done = 0;
  if (ck) {
    if ((rc = ensure_crc(c))) return rc;
    for (auto& v : c->last_crc) v = 0;
    c->last_crc_len = 0;
  }
  SlotRing ring(c, [&](int q) {
    if (ck) {
      const uint64_t* h = static_cast<const uint64_t*>(c->slots[q].crc_out.h.p);
      for (int ty = 0; ty < kCrcTypes; ty++) {
        if (!(ck & (1 << ty))) continue;
        const CrcSpec sp = crc_spec(ty);
        c->last_crc[ty] = ck_done == 0 ? h[ty] : crc_combine(c->crc_host->xp8[ty], c->last_crc[ty], h[ty], ck_len[q], sp.poly, sp.bits);
      }
      ck_done += ck_len[q];
      c->last_crc_len = ck_done;
    }
    retire(inflight[q]);
  });
  for (int64_t b0 = 0; b0 < nall; b0 += chunk) {
    if ((rc = ring.acquire())) return rc;
    const int si = ring.si;
    Slot& s = c->slots[si];
    EncChunk ch;
    ch.b0 = b0; ch.nb = std::min(chunk, nall - b0); ch.s = &s; ch.pitch = pitch;
    const int64_t off = b0 * bs, bytes = std::min(len - off, ch.nb * bs);
    ch.nfull = bytes / bs; ch.tail = bytes % bs;
    if ((rc = s.out.ensure(static_cast<size_t>(ch.nb * std::max(c->m, 1) * pitch)))) return rc;
    if ((rc = s.dig.d.ensure(static_cast<size_t>(ch.nb * c->n * 32)))) return rc;
    Staged sg;
    if ((rc = stage(s, off, bytes, &sg))) return rc;
    if ((rc = s.dig.h.ensure(static_cast<size_t>(ch.nb * c->n * 32)))) return rc;
    ch.st = s.st;
    ch.d_src = sg.obj; ch.d_src_tail = ch.d_src + ch.nfull * bs;
    ch.d_out = static_cast<uint8_t*>(s.out.p); ch.d_out_tail = ch.d_out + ch.nfull * c->m * pitch;
    ch.h_dig = static_cast<const uint8_t*>(s.dig.h.p); ch.h_dig_tail = ch.h_dig + ch.nfull * c->n * 32;
    if ((rc = encode_device_locked(c, sg.obj, bytes, static_cast<uint8_t*>(s.out.p), pitch, static_cast<uint8_t*>(s.dig.d.p), s.st)))
      return rc;
    if (ck) {
      if ((rc = s.crc_out.ensure(kCrcTypes * sizeof(uint64_t)))) return rc;
      if ((rc = checksums_enqueue(c, sg.ck, sg.ck_len, ck, s.crc_part, static_cast<uint64_t*>(s.crc_out.d.p), s.st))) return rc;
      MEC_CUDA_OK(s.crc_out.download(kCrcTypes * sizeof(uint64_t), s.st));
      ck_len[si] = sg.ck_len;
    }
    if ((rc = enqueue(ch))) return rc;
    inflight[si] = ch;
    ring.submitted();
  }
  if ((rc = ring.finish())) return rc;
  c->st_blocks_encoded += nall;
  return MEC_OK;
}

extern "C" int mec_encode_blocks(mec_codec* c, const uint8_t* src, int64_t len, uint8_t* parity, uint8_t* digests) {
  NvtxRange nvtx("mec_encode_blocks");
  if (!c || len < 0) return MEC_ERR_INVALID_ARGUMENT;
  int rc = require_streaming(c);
  if (rc) return rc;
  if (len == 0) {  // cmd/erasure-coding.go:78-80
    reset_last_checksums(c);
    return MEC_OK;
  }
  if (c->S() >= (1ll << 31)) return MEC_ERR_UNSUPPORTED;
  std::lock_guard<std::mutex> lk(c->mu);
  MEC_CUDA_OK(cudaSetDevice(c->device));
  const int64_t S = c->S();
  rc = encode_pipeline(
      c, len, plain_stage(c, src),
      [&](const EncChunk& ch) -> int {
        Slot& s = *ch.s;
        if (c->m > 0 && ch.nfull > 0)
          MEC_CUDA_OK(cudaMemcpy2DAsync(parity + ch.b0 * c->m * S, static_cast<size_t>(S), s.out.p, static_cast<size_t>(ch.pitch),
                                        static_cast<size_t>(S), static_cast<size_t>(ch.nfull * c->m), cudaMemcpyDeviceToHost, s.st));
        if (c->m > 0 && ch.tail > 0) {
          const int64_t St = ceil_frac(ch.tail, c->k);
          MEC_CUDA_OK(cudaMemcpy2DAsync(parity + (ch.b0 + ch.nfull) * c->m * S, static_cast<size_t>(S),
                                        static_cast<uint8_t*>(s.out.p) + ch.nfull * c->m * ch.pitch, static_cast<size_t>(ch.pitch),
                                        static_cast<size_t>(St), static_cast<size_t>(c->m), cudaMemcpyDeviceToHost, s.st));
        }
        MEC_CUDA_OK(cudaMemcpyAsync(digests + ch.b0 * c->n * 32, s.dig.d.p, static_cast<size_t>(ch.nb * c->n * 32),
                                    cudaMemcpyDeviceToHost, s.st));
        return MEC_OK;
      },
      [](const EncChunk&) {});
  if (rc) return rc;
  c->st_d2h += ceil_frac(len, c->block_size) * (c->m * S + c->n * 32);
  return MEC_OK;
}

// a train of independent copies as few driver calls (CUDA 12.8 cudaMemcpyBatchAsync, at most kMaxBatchCopies copies each);
// MEC_NO_BATCH_COPY=1: one call per copy.  A merged GET stages k frames per block; merged GETs of a few hundred blocks whose
// frames all went through ONE call of thousands of copies ended in an unspecified launch failure on an H100, while the same
// batches staged by the gather kernel or by one call per copy did not (tests/test_gpu_batcher.py, get-dma-depth0).
constexpr size_t kMaxBatchCopies = 256;
static int copy_batch(std::vector<void*>& dsts, std::vector<void*>& srcs, std::vector<size_t>& sizes, cudaStream_t st) {
  if (dsts.empty()) return MEC_OK;
  static const bool no_batch = getenv("MEC_NO_BATCH_COPY") != nullptr;
  if (!no_batch && dsts.size() > 1) {
    cudaMemcpyAttributes at = {};
    at.srcAccessOrder = cudaMemcpySrcAccessOrderStream;
    size_t idx0 = 0, fail = 0, done = 0;
    cudaError_t e = cudaSuccess;
    for (; done < dsts.size() && e == cudaSuccess; done += kMaxBatchCopies) {
      const size_t cnt = std::min(kMaxBatchCopies, dsts.size() - done);
      e = cudaMemcpyBatchAsync(dsts.data() + done, srcs.data() + done, sizes.data() + done, cnt, &at, &idx0, 1, &fail, st);
    }
    if (e == cudaSuccess) return MEC_OK;
    if (done > kMaxBatchCopies) {  // part of the train is already queued
      set_last_error(std::string("cudaMemcpyBatchAsync: ") + cudaGetErrorString(e));
      return MEC_ERR_CUDA;
    }
    cudaGetLastError();  // older driver: fall through to separate calls
  }
  for (size_t i = 0; i < dsts.size(); i++) MEC_CUDA_OK(cudaMemcpyAsync(dsts[i], srcs[i], sizes[i], cudaMemcpyDefault, st));
  return MEC_OK;
}

struct CopyList {
  std::vector<void*> dsts, srcs;
  std::vector<size_t> sizes;
  void add(void* d, const void* s, int64_t n) {
    if (n <= 0) return;
    dsts.push_back(d); srcs.push_back(const_cast<void*>(s)); sizes.push_back(static_cast<size_t>(n));
  }
  int flush(cudaStream_t st) {
    const int rc = copy_batch(dsts, srcs, sizes, st);
    dsts.clear(); srcs.clear(); sizes.clear();
    return rc;
  }
};
// chunks of at most this many erasure blocks move as ONE batched copy call per direction instead of one 2-D copy per shard:
// a small GetObject is two driver calls instead of two dozen (the driver lock is what concurrent small requests queue on)
constexpr int64_t kBatchedCopyBlocks = 8;

// Frame sinks of Erasure.Encode.  files[i] is the part.N image of drive i: ([32 B digest][shard bytes])* with full frames
// of 32 + S bytes and one short last frame.  Everything that is bulk moves by DMA straight from device memory into the
// caller's frames (2-D copies: one row per erasure block); only the 32-byte digests go through a pinned staging buffer and
// are scattered by the host while the next chunks are in flight.  No pageable temporaries, no assembly memcpy of shard bytes.
//   parity drives:  frames of drive k+j come from the kernel's parity rows
//   data drives:    with_data = true copies the data shards back from the staged object bytes (the device already holds
//                   them); false leaves the data part to the caller (mec_encode_sg: the writer emits the digest followed
//                   by the slice of its own source buffer, as streamingBitrotWriter.Write does — no copy anywhere)
static int frames_enqueue(mec_codec* c, const EncChunk& ch, uint8_t* const* files, bool with_data, uint8_t* data_digests, CopyList* list = nullptr) {
  const int k = c->k, m = c->m;
  const int64_t bs = c->block_size, S = c->S(), fstride = 32 + S;
  cudaStream_t st = ch.st;
  const int64_t per_t = ch.tail > 0 ? ceil_frac(ch.tail, k) : 0;
  for (int j = 0; j < m; j++) {
    uint8_t* f = files[k + j];
    if (!f) continue;
    f += ch.b0 * fstride + 32;
    if (list) {
      for (int64_t b = 0; b < ch.nfull; b++) list->add(f + b * fstride, ch.d_out + (b * m + j) * ch.pitch, S);
      if (ch.tail > 0) list->add(f + ch.nfull * fstride, ch.d_out_tail + j * ch.pitch, per_t);
    } else {
      if (ch.nfull > 0)
        MEC_CUDA_OK(cudaMemcpy2DAsync(f, static_cast<size_t>(fstride), ch.d_out + j * ch.pitch,
                                      static_cast<size_t>(m * ch.pitch), static_cast<size_t>(S), static_cast<size_t>(ch.nfull),
                                      cudaMemcpyDeviceToHost, st));
      if (ch.tail > 0)
        MEC_CUDA_OK(cudaMemcpyAsync(f + ch.nfull * fstride, ch.d_out_tail + j * ch.pitch,
                                    static_cast<size_t>(per_t), cudaMemcpyDeviceToHost, st));
    }
    c->st_d2h += ch.nfull * S + per_t;
  }
  if (with_data) {
    for (int i = 0; i < k; i++) {
      uint8_t* f = files[i];
      if (!f) continue;
      f += ch.b0 * fstride + 32;
      const int64_t w = std::max<int64_t>(0, std::min(S, bs - static_cast<int64_t>(i) * S));  // Split: the last shard is short, the rest is zero padding
      if (list) {
        for (int64_t b = 0; b < ch.nfull; b++) list->add(f + b * fstride, ch.d_src + b * bs + static_cast<int64_t>(i) * S, w);
      } else if (ch.nfull > 0 && w > 0) {
        MEC_CUDA_OK(cudaMemcpy2DAsync(f, static_cast<size_t>(fstride), ch.d_src + static_cast<int64_t>(i) * S,
                                      static_cast<size_t>(bs), static_cast<size_t>(w), static_cast<size_t>(ch.nfull), cudaMemcpyDeviceToHost, st));
      }
      if (ch.tail > 0) {
        const int64_t start = static_cast<int64_t>(i) * per_t, have = std::max<int64_t>(0, std::min(per_t, ch.tail - start));
        if (list) list->add(f + ch.nfull * fstride, ch.d_src_tail + start, have);
        else if (have > 0)
          MEC_CUDA_OK(cudaMemcpyAsync(f + ch.nfull * fstride, ch.d_src_tail + start,
                                      static_cast<size_t>(have), cudaMemcpyDeviceToHost, st));
      }
      c->st_d2h += ch.nfull * w;
    }
  }
  (void)data_digests;
  return MEC_OK;
}

static void frames_retire(mec_codec* c, const EncChunk& ch, uint8_t* const* files, bool with_data, uint8_t* data_digests) {
  const int k = c->k, n = c->n;
  const int64_t bs = c->block_size, S = c->S(), fstride = 32 + S;
  const int64_t per_t = ch.tail > 0 ? ceil_frac(ch.tail, k) : 0;
  for (int64_t b = 0; b < ch.nb; b++) {
    const bool is_tail = b >= ch.nfull;
    for (int i = 0; i < n; i++) {
      const uint8_t* dg = is_tail ? ch.h_dig_tail + i * 32 : ch.h_dig + (b * n + i) * 32;
      if (data_digests && i < k) memcpy(data_digests + ((ch.b0 + b) * k + i) * 32, dg, 32);
      uint8_t* f = files ? files[i] : nullptr;
      if (!f || (i < k && !with_data)) continue;
      f += (ch.b0 + b) * fstride;
      memcpy(f, dg, 32);  // hash first, then the shard (cmd/bitrot-streaming.go:60,65)
      if (i < k) {        // Split's zero padding behind the object bytes (cmd/erasure-coding.go:81)
        const int64_t per = is_tail ? per_t : S, blen = is_tail ? ch.tail : bs;
        const int64_t have = std::max<int64_t>(0, std::min(per, blen - static_cast<int64_t>(i) * per));
        if (have < per) memset(f + 32 + have, 0, static_cast<size_t>(per - have));
      }
    }
  }
}

// a chunk's digests into its slot's pinned staging (scattered by frames_retire) and its frames into `files` (frames_enqueue)
static int frames_enqueue_chunk(mec_codec* c, const EncChunk& ch, uint8_t* const* files, bool with_data, uint8_t* data_digests) {
  if (ch.nb <= kBatchedCopyBlocks) {  // a small object: digests and every frame piece in ONE batched copy call
    CopyList list;
    list.add(ch.s->dig.h.p, ch.s->dig.d.p, ch.nb * c->n * 32);
    const int e = frames_enqueue(c, ch, files, with_data, data_digests, &list);
    return e ? e : list.flush(ch.st);
  }
  MEC_CUDA_OK(ch.s->dig.download(static_cast<size_t>(ch.nb * c->n * 32), ch.st));
  return frames_enqueue(c, ch, files, with_data, data_digests);
}

static int64_t encode_frames(mec_codec* c, const uint8_t* src, int64_t len, uint8_t* const* files, bool with_data,
                             uint8_t* data_digests, int write_quorum, const char* what) {
  NvtxRange nvtx(what);
  if (!c || len < 0 || !files) return MEC_ERR_INVALID_ARGUMENT;
  int online = 0;
  for (int i = 0; i < c->n; i++) online += files[i] != nullptr;
  if (online < write_quorum) return MEC_ERR_WRITE_QUORUM;  // cmd/erasure-encode.go:59-65
  if (len == 0) {
    reset_last_checksums(c);
    return 0;
  }
  int rc = require_streaming(c);
  if (rc) return rc;
  if (c->S() >= (1ll << 31)) return MEC_ERR_UNSUPPORTED;
  std::lock_guard<std::mutex> lk(c->mu);
  MEC_CUDA_OK(cudaSetDevice(c->device));
  rc = encode_pipeline(
      c, len, plain_stage(c, src),
      [&](const EncChunk& ch) { return frames_enqueue_chunk(c, ch, files, with_data, data_digests); },
      [&](const EncChunk& ch) { frames_retire(c, ch, files, with_data, data_digests); });
  return rc ? rc : len;
}

// Erasure.Encode + streaming bitrot writers (cmd/erasure-encode.go:69, cmd/bitrot-streaming.go:44-75): complete part.N images.
extern "C" int64_t mec_encode(mec_codec* c, const uint8_t* src, int64_t len, uint8_t* const* files, int write_quorum) {
  return encode_frames(c, src, len, files, true, nullptr, write_quorum, "mec_encode");
}

// Scatter-gather form of the same call: the k data shards stay where Split left them — inside `src` — and only what the GPU
// produced comes back: complete frames for the parity drives (files[k..n), NULL = offline) and the digests of the data shards
// ([block][k][32]).  files[0..k) are only tested for NULL (offline writers count against the quorum).
extern "C" int64_t mec_encode_sg(mec_codec* c, const uint8_t* src, int64_t len, uint8_t* const* files, uint8_t* data_digests,
                                 int write_quorum) {
  if (!data_digests) return MEC_ERR_INVALID_ARGUMENT;
  return encode_frames(c, src, len, files, false, data_digests, write_quorum, "mec_encode_sg");
}

// ------------------------------------------------------------------------------------------------
// reconstruct over frames (host)
struct FrameGeom {
  int64_t nblocks, S, last_len;
  int64_t file_bytes() const { return nblocks <= 0 ? 0 : (nblocks - 1) * (32 + S) + 32 + last_len; }
  // frames are staged on the device at a 16-byte aligned pitch so that every TMA row is aligned
  int64_t dpitch() const { return round_up(32 + S, 16); }
  int64_t dev_bytes() const { return nblocks * dpitch() + 512; }
};

// host frames ([32+S] stride, last frame possibly short) -> device frames at pitch g.dpitch()
static int stage_frames(const uint8_t* host, void* dev, const FrameGeom& g, cudaStream_t st) {
  const int64_t nfull = (g.last_len == g.S) ? g.nblocks : g.nblocks - 1;
  if (nfull > 0)
    MEC_CUDA_OK(cudaMemcpy2DAsync(dev, static_cast<size_t>(g.dpitch()), host, static_cast<size_t>(32 + g.S),
                                  static_cast<size_t>(32 + g.S), static_cast<size_t>(nfull), cudaMemcpyHostToDevice, st));
  if (nfull < g.nblocks)
    MEC_CUDA_OK(cudaMemcpyAsync(static_cast<uint8_t*>(dev) + nfull * g.dpitch(), host + nfull * (32 + g.S),
                                static_cast<size_t>(32 + g.last_len), cudaMemcpyHostToDevice, st));
  return MEC_OK;
}

// Where the rebuilt / read shards of a range go.
//   frame sink  (Heal, mec_reconstruct_frames): out[i] = frame-layout image of shard i, same geometry as the inputs
//   object sink (Decode): the data shards of every block, cut to the object bytes [lo, hi) and laid end to end in dst —
//                writeDataBlocks (cmd/erasure-utils.go:42) done by the copy engines: one 2-D copy per data shard and chunk
//   transcode sink (data movement between pools, mec_transcode): the data shards of every block re-split on the device into the
//                object bytes of the whole part, encoded by the codec `enc` and written as complete frames of its geometry to enc_files
//   sealed-object sink (mec_decode_sse): the object sink into a DEVICE buffer (dst_dev), and `accepted(si, blocks)` called on the
//                host each time the range's first `blocks` blocks are final, with slot si the one that carried the last of them
struct RangeSink {
  uint8_t* const* out = nullptr;
  uint8_t* dst = nullptr;
  bool dst_dev = false;
  std::function<int(int, int64_t)> accepted;
  mec_codec* enc = nullptr;
  uint8_t* const* enc_files = nullptr;
  int64_t first_block = 0;   // index (within the part) of the range's first block
  int64_t lo = 0, hi = 0;    // wanted part bytes
  int64_t bs = 0, total = 0; // block size, part size
};

// One chunk of the reconstruct pipeline: blocks [b0, b0 + nb) of the range, read through reader set `chosen`.
struct RChunk : DecodePlan {
  int64_t b0 = 0, nb = 0;
  int chosen[kMaxK];
  uint64_t epoch = 0;  // reader-set generation the chunk was submitted under
};

// survivors of a chunk sit in ONE arena per slot at a uniform stride (position t of the reader set at t * stride)
static inline uint8_t* arena_ptr(Slot& s, int64_t stride, int t) { return static_cast<uint8_t*>(s.aux.p) + t * stride; }

// Rebuild `ch.targets` for the chunk from the staged survivor frames.  d_out rows: (b*r + q); digests [b][k + r]; flags [b][k].
// raw[t] (optional): position t holds rows of a verified whole-file reader laid into frame slots, with no digest to check — its
// expected-digest pointer is null, so the kernel leaves its flags at 0.
static int launch_reconstruct(mec_codec* c, const FrameGeom& g, const RChunk& ch, Slot& s, int64_t stride, const uint8_t* rows,
                              int64_t pitch, bool hash_outputs, const bool* raw = nullptr) {
  const int k = c->k, r = ch.r;
  FusedDesc d;
  d.k = k; d.r = r; d.coef = rows; d.static_encode = false; d.contiguous = false; d.hash_outputs = hash_outputs;
  d.key = kMagicKey; d.out_pitch = pitch; d.expect_block_stride = g.dpitch(); d.in_block_stride = g.dpitch();
  // the range's short last block (if this chunk holds it) is a second launch with its own shard length
  const bool has_short = (ch.b0 + ch.nb == g.nblocks) && g.last_len != g.S;
  const int64_t nfull = has_short ? ch.nb - 1 : ch.nb;
  if (has_short && nfull > 0 && c->eng->small_ok(c->opt, ch.nb)) {  // one launch: the last block carries its own shard length
    d.nblocks = ch.nb;
    d.S = static_cast<int32_t>(g.S);
    d.tail_block = nfull; d.tail_S = static_cast<int32_t>(g.last_len);
    for (int t = 0; t < k; t++) {
      const uint8_t* base = arena_ptr(s, stride, t);
      d.map_base[t] = base; d.map_len[t] = stride; d.expect_ptr[t] = (raw && raw[t]) ? nullptr : base; d.in_ptr[t] = base + 32;
    }
    d.out = static_cast<uint8_t*>(s.out.p);
    d.digests = static_cast<uint8_t*>(s.dig.d.p);
    d.corrupt = static_cast<uint8_t*>(s.flags.d.p);
    return c->eng->launch_fused(d, c->opt, s.st);
  }
  for (int pass = 0; pass < 2; pass++) {
    const int64_t first = pass == 0 ? 0 : nfull;
    const int64_t nb = pass == 0 ? nfull : ch.nb - nfull;
    if (nb <= 0) continue;
    d.nblocks = nb;
    d.S = static_cast<int32_t>(pass == 0 ? g.S : g.last_len);
    for (int t = 0; t < k; t++) {
      const uint8_t* base = arena_ptr(s, stride, t) + first * g.dpitch();
      d.map_base[t] = base;
      d.map_len[t] = stride - first * g.dpitch();
      d.expect_ptr[t] = (raw && raw[t]) ? nullptr : base;
      d.in_ptr[t] = base + 32;
    }
    d.out = static_cast<uint8_t*>(s.out.p) + first * r * pitch;
    d.digests = static_cast<uint8_t*>(s.dig.d.p) + first * (k + r) * 32;
    d.corrupt = static_cast<uint8_t*>(s.flags.d.p) + first * k;
    int rc = c->eng->launch_fused(d, c->opt, s.st);
    if (rc) return rc;
  }
  return MEC_OK;
}

// parallelReader.Read's choice of readers (cmd/erasure-decode.go:145-221): the first k alive readers in index order,
// preferred ones first (preferReaders, :92-123)
static int choose_readers(const mec_codec* c, const uint8_t* const* frames, const uint8_t* alive, const uint8_t* prefer, int* chosen) {
  const int k = c->k, n = c->n;
  int nch = 0;
  if (prefer) {
    int order[kMaxShards], next = 0;
    for (int i = 0; i < n; i++) order[i] = i;
    for (int i = 0; i < n; i++) {
      if (!prefer[i] || frames[i] == nullptr) continue;
      if (i == next) { next++; continue; }
      std::swap(order[next], order[i]);
      next++;
    }
    for (int q = 0; q < n && nch < k; q++)
      if (alive[order[q]]) chosen[nch++] = order[q];
    std::sort(chosen, chosen + nch);  // decode rows are defined on ascending shard indices
  } else {
    for (int i = 0; i < n && nch < k; i++)
      if (alive[i]) chosen[nch++] = i;
  }
  return nch;
}

// writeDataBlocks (cmd/erasure-utils.go:42) for data shard i of part block B, whose shards hold `cur` bytes each: the part bytes
// [a, e) it contributes to the wanted bytes [lo, hi) (none when e <= a), found at `off` in the shard.
struct DataSlice { int64_t a, e, off; };
static inline DataSlice data_slice(int64_t B, int i, int64_t cur, int64_t bs, int64_t total, int64_t lo, int64_t hi) {
  const int64_t blo = B * bs, bhi = std::min(blo + bs, total);
  const int64_t slo = blo + static_cast<int64_t>(i) * cur, shi = std::min(slo + cur, bhi);
  const int64_t a = std::max(slo, lo), e = std::min(shi, hi);
  return DataSlice{a, e, a - slo};
}

// device->host copies of one verified-or-not chunk into the object sink (optimistic: a chunk that turns out to hold a corrupt
// frame is redone from the bad block with other readers and its bytes are overwritten before the call returns)
static int emit_object(mec_codec* c, const FrameGeom& g, const RangeSink& sk, const RChunk& ch, Slot& s, int64_t stride, int64_t pitch,
                       CopyList* list = nullptr) {
  const int k = c->k, r = ch.r;
  const int64_t bs = sk.bs, S = g.S, P = g.dpitch();
  const cudaMemcpyKind kind = sk.dst_dev ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost;
  const int64_t d2h = sk.dst_dev ? 0 : 1;  // device-to-device moves are no copy-back
  for (int i = 0; i < k; i++) {
    // device source of data shard i: a staged survivor frame or a rebuilt row
    const uint8_t* base = nullptr;
    int64_t spitch = 0;
    for (int t = 0; t < k && !base; t++)
      if (ch.chosen[t] == i) { base = arena_ptr(s, stride, t) + 32; spitch = P; }
    for (int q = 0; q < r && !base; q++)
      if (ch.targets[q] == i) { base = static_cast<uint8_t*>(s.out.p) + q * pitch; spitch = r * pitch; }
    if (!base) return MEC_ERR_UNEXPECTED;
    // blocks of the chunk: a run of blocks that are wanted in full goes out as one 2-D copy, partial ones one by one
    int64_t run0 = -1;
    auto flush = [&](int64_t run1) -> int {  // blocks [run0, run1) of the chunk, all full and fully wanted
      if (run0 < 0 || run1 <= run0) { run0 = -1; return MEC_OK; }
      const int64_t w = std::max<int64_t>(0, std::min(S, bs - static_cast<int64_t>(i) * S));
      if (w > 0) {
        const int64_t B = sk.first_block + ch.b0 + run0;
        if (list) {
          for (int64_t q = 0; q < run1 - run0; q++)
            list->add(sk.dst + ((B + q) * bs + static_cast<int64_t>(i) * S - sk.lo), base + (run0 + q) * spitch, w);
        } else {
          MEC_CUDA_OK(cudaMemcpy2DAsync(sk.dst + (B * bs + static_cast<int64_t>(i) * S - sk.lo), static_cast<size_t>(bs), base + run0 * spitch,
                                        static_cast<size_t>(spitch), static_cast<size_t>(w), static_cast<size_t>(run1 - run0), kind, s.st));
        }
        c->st_d2h += d2h * w * (run1 - run0);
      }
      run0 = -1;
      return MEC_OK;
    };
    int rc;
    for (int64_t b = 0; b < ch.nb; b++) {
      const int64_t B = sk.first_block + ch.b0 + b;
      const int64_t blo = B * bs, bhi = std::min(blo + bs, sk.total);          // part bytes of this block
      const int64_t cur = (ch.b0 + b == g.nblocks - 1) ? g.last_len : S;       // its shard length
      const bool whole = blo >= sk.lo && bhi <= sk.hi && bhi - blo == bs && cur == S;
      if (whole) { if (run0 < 0) run0 = b; continue; }
      if ((rc = flush(b))) return rc;
      const DataSlice sl = data_slice(B, i, cur, bs, sk.total, sk.lo, sk.hi);
      if (sl.e > sl.a) {
        if (list) list->add(sk.dst + (sl.a - sk.lo), base + b * spitch + sl.off, sl.e - sl.a);
        else MEC_CUDA_OK(cudaMemcpyAsync(sk.dst + (sl.a - sk.lo), base + b * spitch + sl.off, static_cast<size_t>(sl.e - sl.a), kind, s.st));
        c->st_d2h += d2h * (sl.e - sl.a);
      }
    }
    if ((rc = flush(ch.nb))) return rc;
  }
  return list ? list->flush(s.st) : MEC_OK;
}

// rebuilt shards of a chunk -> frame-layout outputs (digest + shard per block)
static int emit_frames(mec_codec* c, const FrameGeom& g, const RangeSink& sk, const RChunk& ch, Slot& s, int64_t pitch, CopyList* list = nullptr) {
  const int k = c->k, r = ch.r;
  const int64_t fstride = 32 + g.S;
  const bool has_short = (ch.b0 + ch.nb == g.nblocks) && g.last_len != g.S;
  const int64_t nfull = has_short ? ch.nb - 1 : ch.nb;
  for (int q = 0; q < r; q++) {
    uint8_t* dst = sk.out[ch.targets[q]];
    if (!dst) continue;
    dst += ch.b0 * fstride;
    if (list) {
      for (int64_t b = 0; b < ch.nb; b++) {
        list->add(dst + b * fstride, static_cast<uint8_t*>(s.dig.d.p) + (b * (k + r) + k + q) * 32, 32);
        list->add(dst + b * fstride + 32, static_cast<uint8_t*>(s.out.p) + (b * r + q) * pitch, (has_short && b == nfull) ? g.last_len : g.S);
      }
      c->st_d2h += nfull * (32 + g.S) + (has_short ? 32 + g.last_len : 0);
      continue;
    }
    if (nfull > 0) {
      MEC_CUDA_OK(cudaMemcpy2DAsync(dst, static_cast<size_t>(fstride), static_cast<uint8_t*>(s.dig.d.p) + (k + q) * 32,
                                    static_cast<size_t>((k + r) * 32), 32, static_cast<size_t>(nfull), cudaMemcpyDeviceToHost, s.st));
      MEC_CUDA_OK(cudaMemcpy2DAsync(dst + 32, static_cast<size_t>(fstride), static_cast<uint8_t*>(s.out.p) + q * pitch,
                                    static_cast<size_t>(r * pitch), static_cast<size_t>(g.S), static_cast<size_t>(nfull), cudaMemcpyDeviceToHost, s.st));
    }
    if (has_short) {
      const int64_t b = nfull;
      MEC_CUDA_OK(cudaMemcpyAsync(dst + b * fstride, static_cast<uint8_t*>(s.dig.d.p) + (b * (k + r) + k + q) * 32, 32, cudaMemcpyDeviceToHost, s.st));
      MEC_CUDA_OK(cudaMemcpyAsync(dst + b * fstride + 32, static_cast<uint8_t*>(s.out.p) + (b * r + q) * pitch, static_cast<size_t>(g.last_len),
                                  cudaMemcpyDeviceToHost, s.st));
    }
    c->st_d2h += nfull * (32 + g.S) + (has_short ? 32 + g.last_len : 0);
  }
  return list ? list->flush(s.st) : MEC_OK;
}

// Transcode sink of one chunk (whole part, so chunk block b is part block ch.b0 + b): the chunk's data shards, read or rebuilt,
// re-split by ONE launch into the object bytes of its blocks in the destination codec's slot `si` (the same index as the source
// slot, whose stream carries everything), then encoded there and queued as destination frames like mec_encode's.  *out is what
// frames_retire needs once the chunk is accepted.  The destination block size divides the source's (R = bs / ebs): the re-split
// runs in source blocks, and the chunk's object bytes are destination blocks [ch.b0 * R, ...), the part's short last one included.
static_assert(kMaxK <= kBatchMaxFiles, "ResplitParams::src holds one entry per source data shard");
static int emit_transcode(mec_codec* c, const FrameGeom& g, const RangeSink& sk, const RChunk& ch, int si, int64_t stride,
                          int64_t pitch, EncChunk* out) {
  mec_codec* e = sk.enc;
  Slot& s = c->slots[si];
  Slot& d = e->slots[si];
  const int k = c->k;
  const int64_t bs = sk.bs, bytes = std::min(sk.total - ch.b0 * bs, ch.nb * bs);
  const int64_t ebs = e->block_size, enb = ceil_frac(bytes, ebs), epitch = round_up(e->S(), 16);
  int rc;
  if ((rc = d.src.ensure(static_cast<size_t>(round_up(bytes, 16) + 256)))) return rc;
  if ((rc = d.out.ensure(static_cast<size_t>(enb * std::max(e->m, 1) * epitch)))) return rc;
  if ((rc = d.dig.ensure(static_cast<size_t>(enb * e->n * 32)))) return rc;
  ResplitParams p;
  p.obj = static_cast<uint8_t*>(d.src.p);
  p.arena = static_cast<const uint8_t*>(s.aux.p); p.arena_stride = stride; p.P = g.dpitch();
  p.rebuilt = static_cast<const uint8_t*>(s.out.p); p.pitch = pitch; p.r = ch.r;
  p.bs = bs; p.S = g.S;
  p.nfull = bytes / bs; p.tail = bytes % bs; p.tail_S = ceil_frac(p.tail, k);
  for (int t = 0; t < k; t++)
    if (ch.chosen[t] < k) p.src[ch.chosen[t]] = static_cast<int8_t>(t);
  for (int q = 0; q < ch.r; q++) p.src[ch.targets[q]] = static_cast<int8_t>(-1 - q);
  transcode_resplit_kernel<<<dim3(static_cast<unsigned>(ch.nb), static_cast<unsigned>(k)), 128, 0, s.st>>>(p);
  MEC_CUDA_OK(cudaGetLastError());
  c->eng->count_launch();
  if ((rc = encode_device_locked(e, p.obj, bytes, static_cast<uint8_t*>(d.out.p), epitch, static_cast<uint8_t*>(d.dig.d.p), s.st))) return rc;
  EncChunk& ec = *out;
  ec = EncChunk{};
  ec.b0 = ch.b0 * (bs / ebs); ec.nb = enb; ec.nfull = bytes / ebs; ec.tail = bytes % ebs; ec.s = &d; ec.pitch = epitch; ec.st = s.st;
  ec.d_src = p.obj; ec.d_src_tail = p.obj + ec.nfull * ebs;
  ec.d_out = static_cast<uint8_t*>(d.out.p); ec.d_out_tail = ec.d_out + ec.nfull * e->m * epitch;
  ec.h_dig = static_cast<const uint8_t*>(d.dig.h.p); ec.h_dig_tail = ec.h_dig + ec.nfull * e->n * 32;
  return frames_enqueue_chunk(e, ec, sk.enc_files, true, nullptr);
}

// Whole-file readers of a call (wholeBitrotReader, cmd/bitrot-whole.go:66-81): a reader hashes its WHOLE shard file on its first
// read, whatever the offset (xlStorage.ReadFile with a verifier, cmd/xl-storage.go:1931-1950).  Verified files stay on the device
// for the whole call: file i at arena + slot_of[i]*fpitch (k positions, fpitch >= round_up(sfs, 16) + 256), -1 = not staged.
struct WholeSet {
  const uint8_t* const* files;  // raw shard files (host), mec_shard_file_size(total) bytes each
  const uint8_t* sums;          // expected digest of file i at + i*64
  const uint8_t* whole;         // n flags: reader i is whole-file; NULL = every reader
  int algo;
  int64_t sfs, fpitch;
  uint8_t* arena;               // device: k * fpitch + 256 bytes
  uint8_t* dig;                 // device: k x 64 digest slots
  uint8_t* hdig;                // pinned host: k x 64
  int slot_of[kMaxShards];
  bool is_whole(int i) const { return !whole || whole[i]; }
};

static int whole_hash_device(mec_codec* c, int algo, const uint8_t* d_data, int64_t pitch, int64_t len, int64_t count,
                             uint8_t* d_out, cudaStream_t st, const WholeStream* streams);

// One round of whole-file verification over the reader set want[0..nwant): the whole-file readers in it that are not staged yet
// are copied into free arena positions and hashed — by ONE launch over the span of positions that holds them (one_launch; verified
// files inside the span are hashed again, one thread per file, so the launch takes no longer), otherwise one launch per file — and
// a reader whose digest does not match is dropped for the rest of the call (errFileCorrupt: alive[i] = 0, corrupt[i] = 1).
// *dropped tells the caller to choose its readers again.  Drains `st`.
static int whole_round(mec_codec* c, WholeSet& w, const int* want, int nwant, uint8_t* alive, uint8_t* corrupt, bool one_launch,
                       cudaStream_t st, bool* dropped) {
  const int k = c->k, n = c->n, ds = mec_digest_size(w.algo);
  *dropped = false;
  bool used[kMaxK] = {};  // positions held by verified files (every one of them is still a chosen reader)
  for (int i = 0; i < n; i++)
    if (w.slot_of[i] >= 0) used[w.slot_of[i]] = true;
  int fresh[kMaxK], nf = 0;
  for (int q = 0; q < nwant; q++) {
    const int i = want[q];
    if (!w.is_whole(i) || w.slot_of[i] >= 0) continue;
    int pos = 0;
    while (pos < k && used[pos]) pos++;
    if (pos == k) return MEC_ERR_UNEXPECTED;
    used[pos] = true;
    w.slot_of[i] = pos;
    fresh[nf++] = i;
    if (w.sfs > 0)
      MEC_CUDA_OK(cudaMemcpyAsync(w.arena + pos * w.fpitch, w.files[i], static_cast<size_t>(w.sfs), cudaMemcpyHostToDevice, st));
    c->st_h2d += w.sfs;
  }
  if (nf == 0) return MEC_OK;
  int rc;
  if (one_launch) {
    int lo = k, hi = -1;
    for (int q = 0; q < nf; q++) { lo = std::min(lo, w.slot_of[fresh[q]]); hi = std::max(hi, w.slot_of[fresh[q]]); }
    if ((rc = whole_hash_device(c, w.algo, w.arena + lo * w.fpitch, w.fpitch, w.sfs, hi - lo + 1, w.dig + lo * 64, st, nullptr))) return rc;
    c->eng->count_launch();
  } else {
    for (int q = 0; q < nf; q++) {  // one launch per newcomer keeps the arena positions arbitrary; these files are few and the hash is serial anyway
      const int pos = w.slot_of[fresh[q]];
      if ((rc = whole_hash_device(c, w.algo, w.arena + pos * w.fpitch, w.fpitch, w.sfs, 1, w.dig + pos * 64, st, nullptr))) return rc;
      c->eng->count_launch();
    }
  }
  MEC_CUDA_OK(cudaMemcpyAsync(w.hdig, w.dig, static_cast<size_t>(k * 64), cudaMemcpyDeviceToHost, st));
  MEC_CUDA_OK(cudaStreamSynchronize(st));
  for (int q = 0; q < nf; q++) {
    const int i = fresh[q];
    if (memcmp(w.hdig + w.slot_of[i] * 64, w.sums + static_cast<size_t>(i) * 64, static_cast<size_t>(ds)) != 0) {
      alive[i] = 0;
      if (corrupt) corrupt[i] = 1;
      c->st_corrupt++;
      w.slot_of[i] = -1;
      *dropped = true;
    }
  }
  return MEC_OK;
}

// Core of Decode / Heal: frames[i] point at the first frame of the range (host).  The range is cut into chunks that run through
// the codec's six slots — while chunk c is in the kernel, chunk c+1 is being staged and chunk c-1 is on its way back — each
// slot with its own stream, survivor arena, output and flag buffers.  Chunks retire in order: the per-frame digest verdicts
// ([block][reader] flags written by the hash threads) are read, and on the first mismatch the failing readers are dropped
// for the rest of the call (parallelReader.Read: p.readers[i] = nil, cmd/erasure-decode.go:196-199), everything submitted
// behind the bad block is discarded and the range resumes AT the bad block with the next readers in order — exactly the
// block-sequential fail-over of the reference, without giving up the pipelining in the common clean case.
// `whole` (optional) makes the readers it flags whole-file readers, the two kinds mixed as parallelReader mixes them: such a
// reader's frames[i] is only tested for NULL, its rows come from the verified file in whole->arena (block sk.first_block + b of
// the range at row b).  A reader set that holds an unverified whole-file reader is verified first (whole_round), and chosen again
// while readers drop — at the first chunk and at the resume after a streaming reader failed.  Whole-file positions are laid into
// the chunk arena on the device, not staged from the host, and carry no per-frame digest.
static int reconstruct_range(mec_codec* c, const uint8_t* const* frames, const FrameGeom& g, const uint8_t* want,
                             int data_only, const RangeSink& sk, uint8_t* corrupt, uint8_t* alive /*n, in/out*/,
                             const uint8_t* prefer = nullptr, bool hash_outputs = true, WholeSet* whole = nullptr) {
  NvtxRange nvtx("mec_reconstruct_range");
  const int k = c->k, n = c->n;
  if (k > kMaxK) return MEC_ERR_UNSUPPORTED;
  MEC_CUDA_OK(cudaSetDevice(c->device));
  SlotDrain drain(c);
  const int64_t fstride = 32 + g.S, P = g.dpitch(), pitch = round_up(g.S, 16);
  // chunk: ~32 MiB of object per chunk keeps short ranges pipelined over several slots; long ranges take larger chunks (up to four
  // times that) because every chunk costs a host round trip when it retires
  int64_t chunk = std::max<int64_t>(1, (32ll << 20) / std::max<int64_t>(1, g.S * k));
  chunk = std::max(chunk, std::min(4 * chunk, g.nblocks / 12));
  if (g.nblocks < 2 * chunk) chunk = std::max<int64_t>(4, ceil_frac(g.nblocks, 4));  // short ranges: ~four pieces, copies overlap (see encode_pipeline)
  // a move from larger source blocks (legacy 10 MiB parts into 1 MiB blocks): one source block already carries R destination blocks
  // and ~3 of them are the 32 MiB above, so a 64 MiB part would be three chunks; at least four keep its copies overlapping
  if (sk.enc && sk.enc->block_size < sk.bs) chunk = std::min(chunk, ceil_frac(g.nblocks, 4));
  if (c->opt.chunk_blocks > 0) chunk = c->opt.chunk_blocks;
  chunk = std::min(chunk, g.nblocks);
  const int64_t stride = round_up(chunk * P + 512, 256);

  RChunk inflight[kSlots];
  EncChunk enc_inflight[kSlots];  // transcode sink: the destination frames of each chunk
  bool busy[kSlots] = {};
  int head = 0, tail = 0, nbusy = 0;  // ring: tail = oldest in flight, head = next free slot
  int64_t next = 0, done = 0;         // next block to submit, blocks accepted so far
  uint64_t epoch = 0;
  int rc;

  auto submit = [&](int si, int64_t b0) -> int {
    Slot& s = c->slots[si];
    RChunk& ch = inflight[si];
    ch.b0 = b0; ch.nb = std::min(chunk, g.nblocks - b0); ch.epoch = epoch;
    int nch = choose_readers(c, frames, alive, prefer, ch.chosen);
    int e;
    // Only the first submit and the first after a resume can meet a newcomer: every other slot is idle then, so the arena
    // positions a round fills are read by no chunk in flight.
    while (whole && nch >= k) {
      bool dropped = false;
      if ((e = whole_round(c, *whole, ch.chosen, k, alive, corrupt, true, s.st, &dropped))) return e;
      if (!dropped) break;
      nch = choose_readers(c, frames, alive, prefer, ch.chosen);
    }
    if ((e = plan_decode(c, ch.chosen, nch, want, data_only, &ch))) return e;
    bool raw[kMaxK] = {};
    WholeFramesParams wp;
    wp.ncols = 0;
    if (whole)
      for (int t = 0; t < k; t++)
        if (whole->is_whole(ch.chosen[t])) {
          raw[t] = true;
          wp.pos[wp.ncols] = static_cast<int8_t>(t);
          wp.file[wp.ncols++] = static_cast<int8_t>(whole->slot_of[ch.chosen[t]]);
        }
    if ((e = s.aux.ensure(static_cast<size_t>(k * stride)))) return e;
    if ((e = s.out.ensure(static_cast<size_t>(ch.nb * std::max(ch.r, 1) * pitch)))) return e;
    if ((e = s.dig.d.ensure(static_cast<size_t>(ch.nb * (k + ch.r) * 32)))) return e;
    if ((e = s.flags.ensure(static_cast<size_t>(ch.nb * k)))) return e;
    FrameGeom sub = g;  // geometry of the chunk: its last block is short only if it is the range's last block
    sub.nblocks = ch.nb;
    sub.last_len = (b0 + ch.nb == g.nblocks) ? g.last_len : g.S;
    // (one contiguous copy per survivor file + a device-side move to the aligned pitch was slower than these 2-D copies on a 2 GiB
    //  GetObject, although a bare copy-engine probe favours contiguous transfers — tools/copy_probe.cu)
    const bool batched = ch.nb <= kBatchedCopyBlocks;
    CopyList list;
    if (batched) {
      for (int t = 0; t < k; t++)
        for (int64_t j = 0; j < ch.nb && !raw[t]; j++)
          list.add(arena_ptr(s, stride, t) + j * P, frames[ch.chosen[t]] + (b0 + j) * fstride, 32 + (j == ch.nb - 1 ? sub.last_len : g.S));
      if ((e = list.flush(s.st))) return e;
    } else {
      for (int t = 0; t < k; t++)
        if (!raw[t] && (e = stage_frames(frames[ch.chosen[t]] + b0 * fstride, arena_ptr(s, stride, t), sub, s.st))) return e;
    }
    c->st_h2d += sub.file_bytes() * (k - wp.ncols);
    if (wp.ncols > 0) {  // whole-file positions: their rows of the chunk's blocks, from the verified files into the frame slots
      wp.arena = static_cast<uint8_t*>(s.aux.p); wp.arena_stride = stride; wp.P = P;
      wp.files = whole->arena; wp.fpitch = whole->fpitch;
      wp.S = g.S; wp.first = sk.first_block + b0; wp.nb = ch.nb; wp.last_len = sub.last_len;
      whole_rows_frames_kernel<<<dim3(static_cast<unsigned>(ch.nb), static_cast<unsigned>(wp.ncols)), 128, 0, s.st>>>(wp);
      MEC_CUDA_OK(cudaGetLastError());
      c->eng->count_launch();
    }
    MEC_CUDA_OK(cudaMemsetAsync(s.flags.d.p, 0, static_cast<size_t>(ch.nb * k), s.st));
    if ((e = launch_reconstruct(c, g, ch, s, stride, ch.rows.data(), pitch, hash_outputs, whole ? raw : nullptr))) return e;
    MEC_CUDA_OK(s.flags.download(static_cast<size_t>(ch.nb * k), s.st));
    if (sk.enc) { if ((e = emit_transcode(c, g, sk, ch, si, stride, pitch, &enc_inflight[si]))) return e; }
    else if (sk.dst) { if ((e = emit_object(c, g, sk, ch, s, stride, pitch, batched ? &list : nullptr))) return e; }
    else if (sk.out) { if ((e = emit_frames(c, g, sk, ch, s, pitch, batched ? &list : nullptr))) return e; }
    return MEC_OK;
  };

  while (done < g.nblocks) {
    while (nbusy < kSlots && next < g.nblocks) {
      if ((rc = submit(head, next))) return rc;
      next += inflight[head].nb;
      busy[head] = true;
      head = (head + 1) % kSlots;
      nbusy++;
    }
    // retire the oldest chunk
    const int si = tail;
    Slot& s = c->slots[si];
    RChunk& ch = inflight[si];
    MEC_CUDA_OK(cudaStreamSynchronize(s.st));
    busy[si] = false;
    tail = (tail + 1) % kSlots;
    nbusy--;
    const uint8_t* fl = static_cast<const uint8_t*>(s.flags.h.p);
    int64_t bad = ch.nb;
    for (int64_t b = 0; b < ch.nb && bad == ch.nb; b++)
      for (int t = 0; t < k; t++)
        if (fl[b * k + t]) { bad = b; break; }
    const int64_t good = bad;  // blocks [b0, b0 + good) are accepted
    if (good > 0 && sk.out) {  // wanted shards that were read are passed through unchanged
      for (int i = 0; i < n; i++) {
        if (!want[i] || !ch.present[i] || !sk.out[i] || sk.out[i] == frames[i]) continue;
        const int64_t bytes = (ch.b0 + good == g.nblocks) ? (g.file_bytes() - ch.b0 * fstride) : good * fstride;
        memcpy(sk.out[i] + ch.b0 * fstride, frames[i] + ch.b0 * fstride, static_cast<size_t>(bytes));
      }
    }
    if (good > 0 && sk.enc) {  // destination digests of the accepted blocks only; a redo rewrites every frame from the bad block on
      EncChunk acc = enc_inflight[si];
      // `good` whole source blocks are good * R full destination blocks; the part's short last destination block is the chunk's
      // last: accepted only with the whole chunk
      if (good < ch.nb) { acc.nb = acc.nfull = good * (sk.bs / sk.enc->block_size); acc.tail = 0; }
      frames_retire(sk.enc, acc, sk.enc_files, true, nullptr);
      sk.enc->st_blocks_encoded += acc.nb;
    }
    c->st_blocks_read += good;
    c->st_shards_rebuilt += good * ch.r;
    done = ch.b0 + good;
    if (good > 0 && sk.accepted && (rc = sk.accepted(si, done))) return rc;
    if (bad < ch.nb) {  // drop every chosen reader that failed at block `bad`, resume there with the next readers
      for (int t = 0; t < k; t++)
        if (fl[bad * k + t]) {
          if (alive[ch.chosen[t]]) c->st_corrupt++;
          alive[ch.chosen[t]] = 0;
          if (corrupt) corrupt[ch.chosen[t]] = 1;
        }
      for (int q = 0; q < kSlots; q++)  // whatever was submitted behind it ran with the old reader set: discard
        if (busy[q]) { MEC_CUDA_OK(cudaStreamSynchronize(c->slots[q].st)); busy[q] = false; }
      head = tail = 0; nbusy = 0;
      next = done;
      epoch++;
    }
  }
  return MEC_OK;
}

extern "C" int mec_reconstruct_device(mec_codec* c, const uint8_t* const* d_frames, int64_t frame_pitch, int64_t nblocks,
                                      const uint8_t* want, int flags, uint8_t* d_out, int64_t out_pitch,
                                      uint8_t* d_digests, uint8_t* d_corrupt, void* stream) {
  if (!c || !d_frames || !want || nblocks < 0) return MEC_ERR_INVALID_ARGUMENT;
  const int data_only = flags & MEC_RECONSTRUCT_DATA_ONLY;
  int rc = require_streaming(c);
  if (rc) return rc;
  if (nblocks == 0) return MEC_OK;
  const int k = c->k, n = c->n;
  if (n > kMaxShards || k > kMaxK) return MEC_ERR_UNSUPPORTED;
  const int64_t S = c->S();
  if ((frame_pitch & 15) || frame_pitch < 32 + S) return MEC_ERR_INVALID_ARGUMENT;
  if (d_corrupt && !d_digests) return MEC_ERR_INVALID_ARGUMENT;  // the digest check runs in the hash threads: no digests, no bitrot verdict
  int chosen[kMaxShards], nch = 0;
  for (int i = 0; i < n && nch < k; i++)
    if (d_frames[i]) chosen[nch++] = i;
  DecodePlan p;
  if ((rc = plan_decode(c, chosen, nch, want, data_only, &p))) return rc;
  std::lock_guard<std::mutex> lk(c->mu);
  MEC_CUDA_OK(cudaSetDevice(c->device));
  FusedDesc d;
  d.k = k; d.r = p.r; d.coef = p.rows.data(); d.static_encode = false; d.contiguous = false;
  d.key = kMagicKey; d.nblocks = nblocks; d.S = static_cast<int32_t>(S);
  d.in_block_stride = frame_pitch; d.expect_block_stride = frame_pitch;
  for (int t = 0; t < k; t++) {
    const uint8_t* base = d_frames[chosen[t]];
    d.map_base[t] = base;
    d.map_len[t] = nblocks * frame_pitch;
    d.expect_ptr[t] = d_corrupt ? base : nullptr;
    d.in_ptr[t] = base + 32;
  }
  d.out = d_out; d.out_pitch = out_pitch; d.digests = d_digests; d.corrupt = d_corrupt;
  d.hash_outputs = !(flags & MEC_RECONSTRUCT_NO_OUTPUT_DIGESTS);
  return c->eng->launch_fused(d, c->opt, static_cast<cudaStream_t>(stream));
}

extern "C" int mec_reconstruct_frames(mec_codec* c, const uint8_t* const* frames, int64_t nblocks, int64_t last_shard_len,
                                      const uint8_t* want, int data_only, uint8_t* const* out, uint8_t* corrupt) {
  if (!c || !frames || !want || !out || nblocks < 0) return MEC_ERR_INVALID_ARGUMENT;
  if (last_shard_len < 0 || last_shard_len > c->S()) return MEC_ERR_INVALID_ARGUMENT;
  int rc = require_streaming(c);
  if (rc) return rc;
  if (c->n > kMaxShards) return MEC_ERR_UNSUPPORTED;
  std::lock_guard<std::mutex> lk(c->mu);
  if (corrupt) memset(corrupt, 0, static_cast<size_t>(c->n));
  if (nblocks == 0) return MEC_OK;
  FrameGeom g{nblocks, c->S(), last_shard_len > 0 ? last_shard_len : c->S()};
  std::vector<uint8_t> alive(c->n);
  for (int i = 0; i < c->n; i++) alive[i] = frames[i] != nullptr;
  RangeSink sk;
  sk.out = out;
  return reconstruct_range(c, frames, g, want, data_only, sk, corrupt, alive.data());
}

extern "C" int64_t mec_decode(mec_codec* c, const uint8_t* const* files, int64_t offset, int64_t length,
                              int64_t total, uint8_t* dst, int* heal_hint) {
  return mec_decode_prefer(c, files, nullptr, offset, length, total, dst, heal_hint);
}

// The blocks Erasure.Decode reads for part bytes [offset, offset + length) of a part of `total` bytes (cmd/erasure-decode.go:
// 251-281): [start_block, last_block], nblocks of them, the last with shards of last_len bytes.
struct ReadRange { int64_t start_block, last_block, nblocks, last_len; };
static ReadRange read_range(const mec_codec* c, int64_t offset, int64_t length, int64_t total) {
  const int64_t bs = c->block_size, S = c->S(), sfs = mec_shard_file_size(c, total);
  ReadRange rr;
  rr.start_block = offset / bs;
  rr.last_block = (offset + length) / bs;
  if ((offset + length) % bs == 0) rr.last_block--;  // blockLength == 0 => loop breaks (:279-281)
  rr.last_block = std::min(rr.last_block, ceil_frac(sfs, S) - 1);
  rr.nblocks = rr.last_block - rr.start_block + 1;
  rr.last_len = std::min(S, sfs - rr.last_block * S);
  return rr;
}

extern "C" int64_t mec_decode_prefer(mec_codec* c, const uint8_t* const* files, const uint8_t* prefer, int64_t offset,
                                     int64_t length, int64_t total, uint8_t* dst, int* heal_hint) {
  NvtxRange nvtx("mec_decode");
  if (heal_hint) *heal_hint = 0;
  if (!c || !files) return MEC_ERR_INVALID_ARGUMENT;
  if (offset < 0 || length < 0) return MEC_ERR_INVALID_ARGUMENT;      // cmd/erasure-decode.go:240-242
  if (offset + length > total) return MEC_ERR_INVALID_ARGUMENT;       // :243-245
  if (length == 0) return 0;                                          // :247-249
  if (!dst) return MEC_ERR_INVALID_ARGUMENT;
  int rc = require_streaming(c);
  if (rc) return rc;
  std::lock_guard<std::mutex> lk(c->mu);
  const int k = c->k, n = c->n;
  const int64_t bs = c->block_size, S = c->S();
  const ReadRange rr = read_range(c, offset, length, total);
  const FrameGeom g{rr.nblocks, S, rr.last_len};
  // writeDataBlocks (cmd/erasure-utils.go:42): a block whose k shards hold fewer bytes than asked of it is ErrShortData
  // (every block but the part's last holds k*S >= block_size bytes, so only that one can fall short)
  if (static_cast<int64_t>(k) * g.last_len < std::min(offset + length, total) - rr.last_block * bs) return MEC_ERR_SHORT_DATA;
  const int64_t fstride = 32 + S, foff = rr.start_block * fstride;
  std::vector<const uint8_t*> in(n);
  std::vector<uint8_t> alive(n), want(n, 0), corrupt(n, 0);
  for (int i = 0; i < n; i++) { in[i] = files[i] ? files[i] + foff : nullptr; alive[i] = files[i] != nullptr; }
  for (int i = 0; i < k; i++) want[i] = 1;
  RangeSink sk;
  sk.dst = dst; sk.first_block = rr.start_block; sk.lo = offset; sk.hi = offset + length; sk.bs = bs; sk.total = total;
  // GetObject only consumes the data bytes of the rebuilt shards: their digests are not computed
  rc = reconstruct_range(c, in.data(), g, want.data(), 1, sk, corrupt.data(), alive.data(), prefer, false);
  if (rc) return rc;
  if (heal_hint)
    for (int i = 0; i < n; i++)
      if (corrupt[i]) *heal_hint = MEC_ERR_FILE_CORRUPT;
  return length;
}

// Erasure.Heal (cmd/erasure-decode.go:317).  Like the reference it reports bitrot met on the way: when a source reader failed
// its digest the stale shards are still rebuilt from the others and written, and the call returns MEC_ERR_FILE_CORRUPT
// (Heal's `derr`, :338-341,366 — healObject aborts the part on it, cmd/erasure-healing.go:603-608); corrupt[i] names the readers.
extern "C" int mec_heal_prefer(mec_codec* c, const uint8_t* const* files, const uint8_t* prefer, int64_t total,
                               uint8_t* const* out_files, uint8_t* corrupt) {
  NvtxRange nvtx("mec_heal");
  if (!c || !files || !out_files) return MEC_ERR_INVALID_ARGUMENT;
  if (corrupt) memset(corrupt, 0, static_cast<size_t>(c->n));
  int rc = require_streaming(c);
  if (rc) return rc;
  if (total <= 0) return MEC_OK;
  std::lock_guard<std::mutex> lk(c->mu);
  const int n = c->n;
  const int64_t S = c->S(), sfs = mec_shard_file_size(c, total);
  FrameGeom g;
  g.nblocks = ceil_frac(total, c->block_size);
  g.S = S;
  g.last_len = sfs - (g.nblocks - 1) * S;
  std::vector<uint8_t> alive(n), want(n, 0), bad(n, 0);
  for (int i = 0; i < n; i++) { alive[i] = files[i] != nullptr; want[i] = out_files[i] != nullptr; }
  RangeSink sk;
  sk.out = out_files;
  rc = reconstruct_range(c, files, g, want.data(), 0, sk, bad.data(), alive.data(), prefer);
  if (rc) return rc;
  bool any = false;
  for (int i = 0; i < n; i++) { any |= bad[i] != 0; if (corrupt) corrupt[i] = bad[i]; }
  return any ? MEC_ERR_FILE_CORRUPT : MEC_OK;
}
extern "C" int mec_heal(mec_codec* c, const uint8_t* const* files, int64_t total, uint8_t* const* out_files) {
  return mec_heal_prefer(c, files, nullptr, total, out_files, nullptr);
}

// Data movement between pools (decommissionObject / rebalanceObject, cmd/erasure-server-pool-decom.go:605,
// cmd/erasure-server-pool-rebalance.go:848): Erasure.Decode of a whole part on `src` piped into Erasure.Encode on `dst`.  The
// reconstruct pipeline of mec_decode_prefer runs with the transcode sink, so the object bytes never leave the device: each chunk
// is read, verified (and rebuilt where readers are missing), re-split, encoded and written out as dst's frames on one stream.
// dst's block size may be a whole fraction of src's (a legacy blockSizeV1 = 10 MiB part re-PUT with blockSizeV2 = 1 MiB blocks,
// cmd/object-api-common.go:34, cmd/storage-datatypes.go:393): chunks still run in source blocks, each re-split into R = src / dst
// destination blocks.
extern "C" int64_t mec_transcode(mec_codec* src, const uint8_t* const* files, const uint8_t* prefer, int64_t total,
                                 mec_codec* dst, uint8_t* const* out_files, int write_quorum, int* heal_hint) {
  NvtxRange nvtx("mec_transcode");
  if (heal_hint) *heal_hint = 0;
  // one handle cannot be both ends: the source slots hold the survivors while the destination slots hold the re-split bytes
  if (!src || !dst || src == dst || !files || !out_files || total < 0) return MEC_ERR_INVALID_ARGUMENT;
  if (src->block_size % dst->block_size != 0 || src->device != dst->device || src->algo != MEC_HIGHWAYHASH256S ||
      dst->algo != MEC_HIGHWAYHASH256S)
    return MEC_ERR_UNSUPPORTED;
  int online = 0;
  for (int i = 0; i < dst->n; i++) online += out_files[i] != nullptr;
  if (online < write_quorum) return MEC_ERR_WRITE_QUORUM;  // cmd/erasure-encode.go:59-65
  if (total == 0) return 0;
  if (src->k > kMaxK || src->n > kMaxShards || dst->S() >= (1ll << 31)) return MEC_ERR_UNSUPPORTED;
  int rc;
  if ((rc = require_streaming(src)) || (rc = require_streaming(dst))) return rc;
  std::scoped_lock lk(src->mu, dst->mu);  // two threads moving parts in opposite directions lock in the same order
  const int n = src->n;
  const int64_t S = src->S(), sfs = mec_shard_file_size(src, total);
  FrameGeom g;
  g.nblocks = ceil_frac(total, src->block_size);
  g.S = S;
  g.last_len = sfs - (g.nblocks - 1) * S;
  std::vector<uint8_t> alive(n), want(n, 0), corrupt(n, 0);
  for (int i = 0; i < n; i++) alive[i] = files[i] != nullptr;
  for (int i = 0; i < src->k; i++) want[i] = 1;
  RangeSink sk;
  sk.enc = dst; sk.enc_files = out_files; sk.hi = total; sk.bs = src->block_size; sk.total = total;
  // as mec_decode_prefer: the rebuilt data shards are consumed, not stored, so they are not hashed
  rc = reconstruct_range(src, files, g, want.data(), 1, sk, corrupt.data(), alive.data(), prefer, false);
  if (rc) return rc;
  if (heal_hint)
    for (int i = 0; i < n; i++)
      if (corrupt[i]) *heal_hint = MEC_ERR_FILE_CORRUPT;
  return total;
}

// ------------------------------------------------------------------------------------------------
// Server-side encryption: DARE 2.0 packages (minio/sio, AES-256-GCM, dare.cuh).  A call's key schedule and H powers live on the
// device only until it returns.
constexpr int64_t kPkg = kDarePkg, kEPkg = kDareEPkg;
constexpr int64_t kDareMaxPackages = int64_t{1} << 32;  // sequence numbers are uint32 (sio's maxPackageCount)

extern "C" int64_t mec_dare_encrypted_size(int64_t n) {
  if (n < 0 || n > kDareMaxPackages * kPkg) return MEC_ERR_INVALID_ARGUMENT;
  return (n / kPkg) * kEPkg + (n % kPkg ? n % kPkg + kDareOverhead : 0);
}
extern "C" int64_t mec_dare_decrypted_size(int64_t e) {
  if (e < 0 || e > kDareMaxPackages * kEPkg) return MEC_ERR_INVALID_ARGUMENT;
  const int64_t r = e % kEPkg;
  if (r > 0 && r <= kDareOverhead) return MEC_ERR_INVALID_ARGUMENT;
  return (e / kEPkg) * kPkg + (r ? r - kDareOverhead : 0);
}

// The AES round tables of the codec, built by its first DARE call.  Built to completion before any use: later calls and merged batches
// read them from other (non-blocking) slot streams, with nothing else ordering them after this launch.
static int dare_tables(mec_codec* c, cudaStream_t st) {
  DareState& d = c->dare;
  if (d.tabs_ok) return MEC_OK;
  int rc;
  if ((rc = d.tabs.ensure(sizeof(DareTables)))) return rc;
  dare_tables_kernel<<<1, 256, 0, st>>>(static_cast<DareTables*>(d.tabs.p));
  MEC_CUDA_OK(cudaGetLastError());
  c->eng->count_launch();
  MEC_CUDA_OK(cudaStreamSynchronize(st));
  d.tabs_ok = true;
  return MEC_OK;
}

// The first kDareKeyHead bytes of a stream's DareStreamKeys: its nonce (seal; zero for open), whether it opens ChaCha20-Poly1305
// packages (option "dare_chacha20" >= 1), and its raw key as big-endian words
static void dare_key_head(uint8_t* h, const uint8_t* key, const uint8_t* nonce, int chacha) {
  memset(h, 0, kDareKeyHead);
  if (nonce) memcpy(h, nonce, 12);
  h[kDarePolicy] = chacha >= 1;
  uint32_t* rk = reinterpret_cast<uint32_t*>(h + offsetof(DareStreamKeys, rk));
  for (int i = 0; i < 8; i++)
    rk[i] = (uint32_t(key[4 * i]) << 24) | (uint32_t(key[4 * i + 1]) << 16) | (uint32_t(key[4 * i + 2]) << 8) | key[4 * i + 3];
}

// The key heads in `heads` (pinned, kDareKeyHead bytes each) of `ns` streams go to the device table `dk` on `st`; with `aes`, ONE
// dare_setup_kernel launch completes it with the key schedules and H powers (a ChaCha20 seal needs neither)
static int dare_setup(mec_codec* c, DareStreamKeys* dk, const uint8_t* heads, int64_t ns, cudaStream_t st, bool aes = true) {
  int rc;
  if (aes && (rc = dare_tables(c, st))) return rc;
  MEC_CUDA_OK(cudaMemcpy2DAsync(dk, sizeof(DareStreamKeys), heads, kDareKeyHead, kDareKeyHead, static_cast<size_t>(ns),
                                cudaMemcpyHostToDevice, st));
  if (!aes) return MEC_OK;
  dare_setup_kernel<<<static_cast<unsigned>(ns), kDareThreads, 0, st>>>(static_cast<const DareTables*>(c->dare.tabs.p), dk);
  MEC_CUDA_OK(cudaGetLastError());
  c->eng->count_launch();
  return MEC_OK;
}

// Key schedules and H powers of `ns` streams into c->dare.keys, enqueued on `st`; nonces: seal only.  chacha: the call's value of
// option "dare_chacha20" (a seal at 2 writes the raw keys only).
static int dare_keys(mec_codec* c, int64_t ns, const uint8_t* keys, const uint8_t* nonces, cudaStream_t st, int chacha) {
  DareState& d = c->dare;
  int rc;
  if ((rc = d.keys.ensure(static_cast<size_t>(ns) * sizeof(DareStreamKeys))) || (rc = d.hkeys.ensure(static_cast<size_t>(ns) * kDareKeyHead)))
    return rc;
  uint8_t* h = static_cast<uint8_t*>(d.hkeys.p);
  for (int64_t s = 0; s < ns; s++) dare_key_head(h + s * kDareKeyHead, keys + 32 * s, nonces ? nonces + 12 * s : nullptr, chacha);
  return dare_setup(c, static_cast<DareStreamKeys*>(d.keys.p), h, ns, st, !(nonces && chacha == 2));
}

// Zeroes the key material of the call, device and host, once everything on `st` (and before it) is done with it.
struct DareScrub {
  mec_codec* c;
  int64_t ns;
  cudaStream_t st;
  ~DareScrub() {
    cudaMemsetAsync(c->dare.keys.p, 0, static_cast<size_t>(ns) * sizeof(DareStreamKeys), st);
    cudaStreamSynchronize(st);
    explicit_bzero(c->dare.hkeys.p, static_cast<size_t>(ns) * kDareKeyHead);
  }
};

// ONE launch over n package rows (device table pk) with the streams' keys `k`; open writes status[row].  chacha: a seal is
// ChaCha20-Poly1305 instead of AES-256-GCM; an open is followed by ONE dare_chacha_kernel launch over the same rows, which opens the
// cipher-1 packages of the streams that allow it.
static int dare_launch(mec_codec* c, bool seal, bool chacha, const DareStreamKeys* k, const DarePkg* pk, int64_t n, const uint8_t* in,
                       uint8_t* out, uint8_t* status, cudaStream_t st) {
  if (n <= 0) return MEC_OK;
  const DareTables* t = static_cast<const DareTables*>(c->dare.tabs.p);
  const unsigned g = static_cast<unsigned>(n);
  if (seal && chacha) dare_chacha_kernel<true><<<g, kDareThreads, 0, st>>>(k, pk, in, out, status);
  else if (seal) dare_kernel<true><<<g, kDareThreads, 0, st>>>(t, k, pk, in, out, status);
  else dare_kernel<false><<<g, kDareThreads, 0, st>>>(t, k, pk, in, out, status);
  MEC_CUDA_OK(cudaGetLastError());
  c->eng->count_launch();
  if (!seal && chacha) {
    dare_chacha_kernel<false><<<g, kDareThreads, 0, st>>>(k, pk, in, out, status);
    MEC_CUDA_OK(cudaGetLastError());
    c->eng->count_launch();
  }
  (seal ? c->st_dare_sealed : c->st_dare_opened) += n;
  return MEC_OK;
}
static const DareStreamKeys* dare_call_keys(const mec_codec* c) { return static_cast<const DareStreamKeys*>(c->dare.keys.p); }

static inline DarePkg dare_row(int64_t in_off, int64_t out_off, int64_t ref_off, int64_t len, int64_t seq, int stream, bool final) {
  DarePkg r;
  r.in_off = in_off; r.out_off = out_off; r.ref_off = ref_off;
  r.len = static_cast<int32_t>(len); r.seq = static_cast<uint32_t>(seq); r.stream = stream; r.final = final ? 1 : 0;
  return r;
}

extern "C" int mec_dare_device(mec_codec* c, int op, int64_t nstreams, const uint8_t* keys, const uint8_t* nonces, const uint32_t* seq0,
                               const int64_t* enc_totals, const uint8_t* d_in, const int64_t* in_off, const int64_t* lens, uint8_t* d_out,
                               const int64_t* out_off, uint8_t* status, void* stream) {
  NvtxRange nvtx("mec_dare_device");
  if (!c || (op != MEC_DARE_SEAL && op != MEC_DARE_OPEN) || nstreams < 0 || nstreams > (int64_t{1} << 31) - 1)
    return MEC_ERR_INVALID_ARGUMENT;
  if (nstreams == 0) return MEC_OK;
  const bool seal = op == MEC_DARE_SEAL;
  if (!keys || !seq0 || !in_off || !lens || !out_off || !status || (seal ? !nonces : !enc_totals)) return MEC_ERR_INVALID_ARGUMENT;
  int64_t rows = 0;
  for (int64_t s = 0; s < nstreams; s++) {
    if (in_off[s] < 0 || out_off[s] < 0 || lens[s] < 0 || (lens[s] > 0 && (!d_in || !d_out))) return MEC_ERR_INVALID_ARGUMENT;
    const int64_t np = seal ? ceil_frac(lens[s], kPkg) : ceil_frac(lens[s], kEPkg);
    if (seal && static_cast<int64_t>(seq0[s]) + np > kDareMaxPackages) return MEC_ERR_INVALID_ARGUMENT;
    rows += np;
  }
  std::lock_guard<std::mutex> lk(c->mu);
  int rc;
  if ((rc = ensure_engine(c))) return rc;
  MEC_CUDA_OK(cudaSetDevice(c->device));
  DareState& d = c->dare;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int chacha = c->dare_chacha20.load();
  const size_t tab = static_cast<size_t>(std::max<int64_t>(rows, 1)) * sizeof(DarePkg);
  if ((rc = d.pk.ensure(tab)) || (rc = d.st.ensure(static_cast<size_t>(std::max<int64_t>(rows, 1)))))
    return rc;
  if ((rc = dare_keys(c, nstreams, keys, seal ? nonces : nullptr, st, chacha))) return rc;
  DareScrub scrub{c, nstreams, st};
  DarePkg* t = static_cast<DarePkg*>(d.pk.h.p);
  int64_t w = 0;
  for (int64_t s = 0; s < nstreams; s++) {
    status[s] = 0;
    const int si = static_cast<int>(s);
    if (seal) {  // a stream of lens[s] bytes from sequence number seq0[s]: its last package is final
      const int64_t np = ceil_frac(lens[s], kPkg);
      for (int64_t j = 0; j < np; j++)
        t[w++] = dare_row(in_off[s] + j * kPkg, out_off[s] + j * kEPkg, 0, std::min(kPkg, lens[s] - j * kPkg), seq0[s] + j, si, j == np - 1);
      continue;
    }
    // open: packages from seq0[s] as the stored part size lays them out; a size that is no DARE size, bytes past the part or a
    // package cut short fail the stream (the whole packages before that point are still opened)
    const int64_t D = mec_dare_decrypted_size(enc_totals[s]);
    if (D < 0) { status[s] = static_cast<uint8_t>(-MEC_ERR_NOT_AUTHENTIC); continue; }
    const int64_t npart = ceil_frac(D, kPkg);
    for (int64_t pos = 0, p = seq0[s]; pos < lens[s]; p++) {
      const int64_t plen = p == npart - 1 ? D - p * kPkg : kPkg;
      if (p >= npart || pos + plen + kDareOverhead > lens[s]) { status[s] = static_cast<uint8_t>(-MEC_ERR_NOT_AUTHENTIC); break; }
      t[w++] = dare_row(in_off[s] + pos, out_off[s] + (p - seq0[s]) * kPkg, in_off[s], plen, p, si, p == npart - 1);
      pos += plen + kDareOverhead;
    }
  }
  if (w > 0) {
    MEC_CUDA_OK(d.pk.upload(static_cast<size_t>(w) * sizeof(DarePkg), st));
    if ((rc = dare_launch(c, seal, seal ? chacha == 2 : chacha >= 1, dare_call_keys(c), static_cast<const DarePkg*>(d.pk.d.p), w, d_in, d_out,
                          static_cast<uint8_t*>(d.st.d.p), st)))
      return rc;
    if (!seal) MEC_CUDA_OK(d.st.download(static_cast<size_t>(w), st));
  }
  MEC_CUDA_OK(cudaStreamSynchronize(st));
  if (!seal) {
    const uint8_t* v = static_cast<const uint8_t*>(d.st.h.p);
    for (int64_t r = 0; r < w; r++) {
      uint8_t& o = status[t[r].stream];
      if (v[r] == kDareUnsupported) o = static_cast<uint8_t>(-MEC_ERR_UNSUPPORTED);
      else if (v[r] == kDareNotAuthentic && o == 0) o = static_cast<uint8_t>(-MEC_ERR_NOT_AUTHENTIC);
    }
  }
  int worst = MEC_OK;
  for (int64_t s = 0; s < nstreams; s++) {
    if (status[s] == static_cast<uint8_t>(-MEC_ERR_UNSUPPORTED)) worst = MEC_ERR_UNSUPPORTED;
    else if (status[s] && worst == MEC_OK) worst = MEC_ERR_NOT_AUTHENTIC;
  }
  return worst;
}

// The packages of a sealed stream of `len` plaintext bytes that overlap the ciphertext bytes [off, off + bytes) of an encode chunk
struct DareSpan {
  int64_t p0, p1, np;  // packages [p0, p1], np of them
  int64_t pt0, pt1;    // their plaintext [pt0, pt1)
  int64_t ps;          // the first package that starts in the chunk (p1 + 1: none does)
  int64_t delta, pad;  // ciphertext byte off is delta bytes into package p0, which is sealed pad bytes into the slot so that off
                       // lands 16-byte aligned for the encode
};
static DareSpan dare_span(int64_t len, int64_t off, int64_t bytes) {
  DareSpan d;
  d.p0 = off / kEPkg; d.p1 = (off + bytes - 1) / kEPkg; d.np = d.p1 - d.p0 + 1;
  d.pt0 = d.p0 * kPkg; d.pt1 = std::min(len, (d.p1 + 1) * kPkg);
  d.ps = ceil_frac(off, kEPkg);
  d.delta = off - d.p0 * kEPkg; d.pad = (16 - d.delta % 16) % 16;
  return d;
}

// Seals the packages of `d` on s.st from their plaintext at `pt` (device, plaintext byte d.pt0; 16-byte aligned for the fast
// loads) into s.src, and points the chunk's staged object bytes at the ciphertext and its checksum bytes at the plaintext of the
// packages that start in the chunk, as hash.Reader sees each byte once.  chacha: ChaCha20-Poly1305 packages (option 2).
static int dare_seal_chunk(mec_codec* c, Slot& s, const DareSpan& d, int64_t len, const uint8_t* pt, Staged* o, bool chacha) {
  const int64_t npk = ceil_frac(len, kPkg);
  int e;
  if ((e = s.src.ensure(static_cast<size_t>(d.pad + d.np * kEPkg + 256))) || (e = s.dpk.ensure(static_cast<size_t>(d.np) * sizeof(DarePkg))))
    return e;
  DarePkg* t = static_cast<DarePkg*>(s.dpk.h.p);
  for (int64_t j = 0; j < d.np; j++) {
    const int64_t p = d.p0 + j;
    t[j] = dare_row(j * kPkg, d.pad + j * kEPkg, 0, std::min(kPkg, len - p * kPkg), p, 0, p == npk - 1);
  }
  MEC_CUDA_OK(s.dpk.upload(static_cast<size_t>(d.np) * sizeof(DarePkg), s.st));
  uint8_t* ct = static_cast<uint8_t*>(s.src.p);
  if ((e = dare_launch(c, true, chacha, dare_call_keys(c), static_cast<const DarePkg*>(s.dpk.d.p), d.np, pt, ct, nullptr, s.st))) return e;
  o->obj = ct + d.pad + d.delta;
  o->ck = pt + (d.ps - d.p0) * kPkg;
  o->ck_len = d.ps <= d.p1 ? d.pt1 - d.ps * kPkg : 0;
  return MEC_OK;
}

// EncryptRequest + Erasure.Encode: chunks are whole erasure blocks of the ciphertext.  A chunk stages and seals every package that
// overlaps it (one across a chunk boundary is sealed in both: sealing is deterministic) and encodes its ciphertext unchanged.
// "checksums" covers the plaintext, as hash.Reader sees it: each chunk the packages that start in it.  chacha: the value of option
// "dare_chacha20" the call runs under (2 seals ChaCha20-Poly1305 packages).
static int64_t encode_sse(mec_codec* c, const uint8_t* src, int64_t len, const uint8_t* key, const uint8_t* nonce, uint8_t* const* files,
                          int write_quorum, int chacha) {
  if (!c || len < 0 || !files || !key || !nonce || (len > 0 && !src)) return MEC_ERR_INVALID_ARGUMENT;
  const int64_t E = mec_dare_encrypted_size(len);
  if (E < 0) return E;
  int online = 0;
  for (int i = 0; i < c->n; i++) online += files[i] != nullptr;
  if (online < write_quorum) return MEC_ERR_WRITE_QUORUM;  // cmd/erasure-encode.go:59-65
  if (len == 0) {
    reset_last_checksums(c);
    return 0;
  }
  int rc = require_streaming(c);
  if (rc) return rc;
  if (c->S() >= (1ll << 31)) return MEC_ERR_UNSUPPORTED;
  std::lock_guard<std::mutex> lk(c->mu);
  MEC_CUDA_OK(cudaSetDevice(c->device));
  Slot& s0 = c->slots[0];
  if ((rc = dare_keys(c, 1, key, nonce, s0.st, chacha))) return rc;
  DareScrub scrub{c, 1, s0.st};
  MEC_CUDA_OK(cudaStreamSynchronize(s0.st));  // every slot stream reads the keys
  auto stage = [&](Slot& s, int64_t off, int64_t bytes, Staged* o) -> int {
    const DareSpan d = dare_span(len, off, bytes);
    int e;
    if ((e = s.aux.ensure(static_cast<size_t>(round_up(d.pt1 - d.pt0, 16) + 256)))) return e;
    MEC_CUDA_OK(cudaMemcpyAsync(s.aux.p, src + d.pt0, static_cast<size_t>(d.pt1 - d.pt0), cudaMemcpyHostToDevice, s.st));
    c->st_h2d += d.pt1 - d.pt0;
    return dare_seal_chunk(c, s, d, len, static_cast<const uint8_t*>(s.aux.p), o, chacha == 2);
  };
  rc = encode_pipeline(
      c, E, stage,
      [&](const EncChunk& ch) { return frames_enqueue_chunk(c, ch, files, true, nullptr); },
      [&](const EncChunk& ch) { frames_retire(c, ch, files, true, nullptr); });
  return rc ? rc : len;
}
extern "C" int64_t mec_encode_sse(mec_codec* c, const uint8_t* src, int64_t len, const uint8_t* key, const uint8_t* nonce,
                                  uint8_t* const* files, int write_quorum) {
  NvtxRange nvtx("mec_encode_sse");
  return encode_sse(c, src, len, key, nonce, files, write_quorum, c ? c->dare_chacha20.load() : 0);
}

// Erasure.Decode of the ciphertext range GetDecryptedRange maps the plaintext range to, then DecryptBlocksRequestR, for one part.
// Chunks move their data slices device-to-device into a ciphertext buffer of the range; whenever a prefix of the range is final
// the packages it completes are opened, each once, and their asked-for plaintext is copied back.  chacha: the value of option
// "dare_chacha20" the call runs under (>= 1 opens ChaCha20-Poly1305 packages too).
static int64_t decode_sse(mec_codec* c, const uint8_t* const* files, const uint8_t* prefer, int64_t offset, int64_t length,
                          int64_t enc_total, const uint8_t* key, uint8_t* dst, int* heal_hint, int chacha) {
  if (heal_hint) *heal_hint = 0;
  if (!c || !files || !key || offset < 0 || length < 0 || enc_total < 0) return MEC_ERR_INVALID_ARGUMENT;
  const int64_t D = mec_dare_decrypted_size(enc_total);
  if (D < 0) return MEC_ERR_NOT_AUTHENTIC;  // ObjectInfo.DecryptedSize: errObjectTampered
  if (offset + length > D) return MEC_ERR_INVALID_ARGUMENT;
  if (length == 0) return 0;
  if (!dst) return MEC_ERR_INVALID_ARGUMENT;
  int rc = require_streaming(c);
  if (rc) return rc;
  std::lock_guard<std::mutex> lk(c->mu);
  MEC_CUDA_OK(cudaSetDevice(c->device));
  const int k = c->k, n = c->n;
  const int64_t bs = c->block_size, S = c->S();
  const int64_t npk = ceil_frac(D, kPkg);
  const int64_t p_first = offset / kPkg, p_last = (offset + length - 1) / kPkg, np = p_last - p_first + 1;
  const int64_t eoff = p_first * kEPkg, eend = std::min(enc_total, (p_last + 1) * kEPkg), elen = eend - eoff;
  const ReadRange rr = read_range(c, eoff, elen, enc_total);
  const FrameGeom g{rr.nblocks, S, rr.last_len};
  if (static_cast<int64_t>(k) * g.last_len < eend - rr.last_block * bs) return MEC_ERR_SHORT_DATA;  // as mec_decode_prefer
  DareState& d = c->dare;
  if ((rc = d.ct.ensure(static_cast<size_t>(round_up(elen, 16) + 256))) || (rc = d.pt.ensure(static_cast<size_t>(np * kPkg))) ||
      (rc = d.st.ensure(static_cast<size_t>(np))) ||
      (rc = d.pk.ensure(static_cast<size_t>(np) * sizeof(DarePkg))))
    return rc;
  Slot& s0 = c->slots[0];
  if ((rc = dare_keys(c, 1, key, nullptr, s0.st, chacha))) return rc;
  DareScrub scrub{c, 1, s0.st};
  DarePkg* t = static_cast<DarePkg*>(d.pk.h.p);
  for (int64_t j = 0; j < np; j++) {
    const int64_t p = p_first + j;
    t[j] = dare_row(j * kEPkg, j * kPkg, 0, p == npk - 1 ? D - p * kPkg : kPkg, p, 0, p == npk - 1);
  }
  MEC_CUDA_OK(d.pk.upload(static_cast<size_t>(np) * sizeof(DarePkg), s0.st));
  MEC_CUDA_OK(cudaMemsetAsync(d.st.d.p, 0, static_cast<size_t>(np), s0.st));
  MEC_CUDA_OK(cudaStreamSynchronize(s0.st));
  uint8_t* ct = static_cast<uint8_t*>(d.ct.p);
  const uint8_t* pt = static_cast<const uint8_t*>(d.pt.p);
  int64_t opened = 0;
  RangeSink sk;
  sk.dst = ct; sk.dst_dev = true; sk.first_block = rr.start_block; sk.lo = eoff; sk.hi = eend; sk.bs = bs; sk.total = enc_total;
  sk.accepted = [&](int si, int64_t blocks) -> int {
    const int64_t acc = std::min(eend, (rr.start_block + blocks) * bs) - eoff;  // final ciphertext bytes of the range
    const int64_t upto = acc == elen ? np : acc / kEPkg;                        // packages they complete
    if (upto <= opened) return MEC_OK;
    Slot& s = c->slots[si];
    int e;
    if ((e = dare_launch(c, false, chacha >= 1, dare_call_keys(c), static_cast<const DarePkg*>(d.pk.d.p) + opened, upto - opened, ct,
                         static_cast<uint8_t*>(d.pt.p), static_cast<uint8_t*>(d.st.d.p) + opened, s.st)))
      return e;
    const int64_t a = std::max(offset, (p_first + opened) * kPkg), z = std::min(offset + length, (p_first + upto) * kPkg);
    if (z > a) {
      MEC_CUDA_OK(cudaMemcpyAsync(dst + (a - offset), pt + (a - p_first * kPkg), static_cast<size_t>(z - a), cudaMemcpyDeviceToHost, s.st));
      c->st_d2h += z - a;
    }
    opened = upto;
    return MEC_OK;
  };
  const int64_t fstride = 32 + S, foff = rr.start_block * fstride;
  std::vector<const uint8_t*> in(n);
  std::vector<uint8_t> alive(n), want(n, 0), corrupt(n, 0);
  for (int i = 0; i < n; i++) { in[i] = files[i] ? files[i] + foff : nullptr; alive[i] = files[i] != nullptr; }
  for (int i = 0; i < k; i++) want[i] = 1;
  rc = reconstruct_range(c, in.data(), g, want.data(), 1, sk, corrupt.data(), alive.data(), prefer, false);
  if (rc) return rc;  // every slot stream has drained
  if (opened != np) return MEC_ERR_UNEXPECTED;
  MEC_CUDA_OK(cudaMemcpy(d.st.h.p, d.st.d.p, static_cast<size_t>(np), cudaMemcpyDeviceToHost));
  const uint8_t* v = static_cast<const uint8_t*>(d.st.h.p);
  int bad = MEC_OK;
  for (int64_t j = 0; j < np; j++) {
    if (v[j] == kDareUnsupported) bad = MEC_ERR_UNSUPPORTED;
    else if (v[j] != kDareOk && bad == MEC_OK) bad = MEC_ERR_NOT_AUTHENTIC;
  }
  if (bad) {  // failed packages wrote no plaintext: hand out nothing of the range
    memset(dst, 0, static_cast<size_t>(length));
    return bad;
  }
  if (heal_hint)
    for (int i = 0; i < n; i++)
      if (corrupt[i]) *heal_hint = MEC_ERR_FILE_CORRUPT;
  return length;
}
extern "C" int64_t mec_decode_sse(mec_codec* c, const uint8_t* const* files, const uint8_t* prefer, int64_t offset, int64_t length,
                                  int64_t enc_total, const uint8_t* key, uint8_t* dst, int* heal_hint) {
  NvtxRange nvtx("mec_decode_sse");
  return decode_sse(c, files, prefer, offset, length, enc_total, key, dst, heal_hint, c ? c->dare_chacha20.load() : 0);
}

// ------------------------------------------------------------------------------------------------
// Signature V4 streaming payloads (sigv4.cuh): the aws-chunked body of a PutObject is de-framed on the host, header bytes only,
// and every chunk's signature is checked on the device, one thread per chunk.
constexpr int64_t kMaxAwsChunk = 16 << 20;  // maxChunkSize, cmd/streaming-signature-v4.go:260
static_assert(MEC_SIGV4_PAYLOAD == kSigPayload && MEC_SIGV4_TRAILER == kSigTrailer, "sigv4.cuh");

static bool lower_hex64(const uint8_t* s) {
  for (int i = 0; i < 64; i++)
    if (!((s[i] >= '0' && s[i] <= '9') || (s[i] >= 'a' && s[i] <= 'f'))) return false;
  return true;
}

// The call's SigCall into the codec's pinned copy: key states and "date\nscope\n".  False when the head does not fit.
static bool sig_call_host(mec_codec* c, const uint8_t* key, const char* date, const char* scope) {
  const size_t dl = strlen(date), sl = strlen(scope);
  if (dl + sl + 2 > static_cast<size_t>(kSigMaxHead)) return false;
  SigCall* k = static_cast<SigCall*>(c->sig.call.h.p);
  memset(k, 0, sizeof(SigCall));
  sig_key_states(key, k);
  memcpy(k->head, date, dl);
  k->head[dl] = '\n';
  memcpy(k->head + dl + 1, scope, sl);
  k->head[dl + sl + 1] = '\n';
  k->head_len = static_cast<int32_t>(dl + sl + 2);
  return true;
}

// Zeroes the call's key states, device and host, once `st` and the slots' verify streams are done with them.
struct SigScrub {
  mec_codec* c;
  cudaStream_t st;
  ~SigScrub() {
    for (auto& s : c->slots)
      if (s.st2) cudaStreamSynchronize(s.st2);
    cudaMemsetAsync(c->sig.call.d.p, 0, sizeof(SigCall), st);
    cudaStreamSynchronize(st);
    explicit_bzero(c->sig.call.h.p, sizeof(SigCall));
  }
};

// Uploads the call's SigCall on `st` and waits for it: every slot stream reads it
static int sig_call_upload(mec_codec* c, cudaStream_t st) {
  MEC_CUDA_OK(c->sig.call.upload(sizeof(SigCall), st));
  MEC_CUDA_OK(cudaStreamSynchronize(st));
  return MEC_OK;
}

// enqueue: the n rows of the host table `h` (sorted here) to the device table `d` on st, then ONE sigv4_chunk_kernel launch whose
// verdicts follow the n rows in `d`
static int sig_launch(mec_codec* c, SigRow* h, SigRow* d, int64_t n, cudaStream_t st) {
  std::sort(h, h + n, [](const SigRow& x, const SigRow& y) { return x.len > y.len; });
  MEC_CUDA_OK(cudaMemcpyAsync(d, h, static_cast<size_t>(n) * sizeof(SigRow), cudaMemcpyHostToDevice, st));
  SigParams p;
  p.rows = d; p.nrows = n; p.call = static_cast<const SigCall*>(c->sig.call.d.p);
  p.verdict = reinterpret_cast<uint8_t*>(d + n);
  sigv4_chunk_kernel<<<static_cast<unsigned>(ceil_frac(n, kSigThreads)), kSigThreads, 0, st>>>(p);
  MEC_CUDA_OK(cudaGetLastError());
  c->eng->count_launch();
  c->st_sigv4_chunks += n;
  return MEC_OK;
}
static inline SigRow sig_row(const uint8_t* msg, int64_t len, int64_t out, int32_t kind, const uint8_t* prev, const uint8_t* claim) {
  SigRow r;
  r.msg = msg; r.len = len; r.out = out; r.kind = kind; r.pad = 0;
  memcpy(r.prev, prev, 64);
  memcpy(r.claim, claim, 64);
  return r;
}

static int sig_ensure(mec_codec* c) {
  int rc;
  if ((rc = c->sig.call.ensure(sizeof(SigCall)))) return rc;
  return MEC_OK;
}

extern "C" int mec_chunk_signatures_device(mec_codec* c, const uint8_t* key, const char* date, const char* scope, const uint8_t* d_base,
                                           const int64_t* offsets, const int64_t* lens, const uint8_t* prev, const uint8_t* claimed,
                                           const int32_t* kinds, int64_t count, uint8_t* verdicts, void* stream) {
  NvtxRange nvtx("mec_chunk_signatures_device");
  if (!c || !key || !date || !scope || count < 0 || strlen(date) + strlen(scope) + 2 > static_cast<size_t>(kSigMaxHead))
    return MEC_ERR_INVALID_ARGUMENT;
  if (count == 0) return MEC_OK;
  if (!offsets || !lens || !prev || !claimed || !kinds || !verdicts) return MEC_ERR_INVALID_ARGUMENT;
  for (int64_t i = 0; i < count; i++)
    if (offsets[i] < 0 || lens[i] < 0 || (lens[i] > 0 && !d_base) || (kinds[i] != kSigPayload && kinds[i] != kSigTrailer))
      return MEC_ERR_INVALID_ARGUMENT;
  if (count > (int64_t{1} << 36)) return MEC_ERR_UNSUPPORTED;  // the grid's x dimension
  std::lock_guard<std::mutex> lk(c->mu);
  int rc;
  if ((rc = ensure_engine(c))) return rc;
  MEC_CUDA_OK(cudaSetDevice(c->device));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const size_t tab = static_cast<size_t>(count) * (sizeof(SigRow) + 1);
  if ((rc = sig_ensure(c)) || (rc = c->sig.rows.ensure(tab))) return rc;
  sig_call_host(c, key, date, scope);
  SigScrub scrub{c, st};
  if ((rc = sig_call_upload(c, st))) return rc;
  SigRow* h = static_cast<SigRow*>(c->sig.rows.h.p);
  for (int64_t i = 0; i < count; i++)
    h[i] = sig_row(d_base + offsets[i], lens[i], i, kinds[i], prev + 64 * i, claimed + 64 * i);
  SigRow* d = static_cast<SigRow*>(c->sig.rows.d.p);
  if ((rc = sig_launch(c, h, d, count, st))) return rc;
  MEC_CUDA_OK(cudaMemcpyAsync(h + count, d + count, static_cast<size_t>(count), cudaMemcpyDeviceToHost, st));
  MEC_CUDA_OK(cudaStreamSynchronize(st));
  memcpy(verdicts, h + count, static_cast<size_t>(count));
  return MEC_OK;
}

// One aws-chunk whose header framed and whose payload is in the body: one signature row
struct AwsChunk {
  int64_t pay, size;  // body offset and length of the payload
  int64_t doff;       // decoded offset of its first payload byte
  const uint8_t* prev;
  const uint8_t* claim;
};
struct ChunkedBody {
  std::vector<AwsChunk> ch;
  std::vector<uint8_t> tmsg;        // trailer mode: the trailer value as signed (with the '\n' readTrailers adds)
  const uint8_t* tclaim = nullptr;  // its claimed signature (NULL: no trailer row)
  int64_t decoded = 0;
};

// bytes.TrimSpace: ASCII white space and the UTF-8 forms of Unicode White_Space
static int space_prefix(const uint8_t* p, int64_t n) {
  if (n >= 1 && (p[0] == ' ' || (p[0] >= '\t' && p[0] <= '\r'))) return 1;
  if (n >= 2 && p[0] == 0xc2 && (p[1] == 0x85 || p[1] == 0xa0)) return 2;
  if (n >= 3 && ((p[0] == 0xe1 && p[1] == 0x9a && p[2] == 0x80) || (p[0] == 0xe3 && p[1] == 0x80 && p[2] == 0x80) ||
                 (p[0] == 0xe2 && p[1] == 0x80 && ((p[2] >= 0x80 && p[2] <= 0x8a) || p[2] == 0xa8 || p[2] == 0xa9 || p[2] == 0xaf)) ||
                 (p[0] == 0xe2 && p[1] == 0x81 && p[2] == 0x9f)))
    return 3;
  return 0;
}
static void trim_space(const uint8_t*& p, int64_t& n) {
  for (int k; n > 0 && (k = space_prefix(p, n)) > 0;) { p += k; n -= k; }
  for (bool more = true; more && n > 0;) {
    more = false;
    for (int k = 1; k <= 3 && k <= n; k++)
      if (space_prefix(p + n - k, k) == k) { n -= k; more = true; break; }
  }
}

// s3ChunkedReader.Read (cmd/streaming-signature-v4.go:264-442) and readTrailers (:445-512) over the body, byte for byte, reading
// header bytes only.  Returns what the serial reader reports once every row recorded in `o` has passed its signature check: MEC_OK,
// a framing error, MEC_ERR_OVERREAD (HardLimitReader, internal/ioutil/hardlimitreader.go:46-56), MEC_ERR_INCOMPLETE_BODY (an
// unexpected EOF, or fewer payload bytes than D: cmd/erasure-object.go:1450-1453) or MEC_ERR_SIGNATURE_MISMATCH (a trailer
// signature that is not 64 bytes long).
static int parse_chunked(const uint8_t* b, int64_t blen, int64_t D, const uint8_t* seed, bool trailer, ChunkedBody* o) {
  int64_t pos = 0;
  const uint8_t* prev = seed;
  for (;;) {
    int64_t size = 0;
    for (;;) {  // hex size digits of either case up to ';' (none: a zero-size chunk)
      if (pos >= blen) return MEC_ERR_INCOMPLETE_BODY;
      const uint8_t x = b[pos++];
      if (x == ';') break;
      int v;
      if (x >= '0' && x <= '9') v = x - '0';
      else if (x >= 'a' && x <= 'f') v = x - 'a' + 10;
      else if (x >= 'A' && x <= 'F') v = x - 'A' + 10;
      else return MEC_ERR_MALFORMED_ENCODING;
      size = size << 4 | v;
      if (size > kMaxAwsChunk) return MEC_ERR_CHUNK_TOO_BIG;
    }
    if (blen - pos < 80) return MEC_ERR_INCOMPLETE_BODY;
    if (memcmp(b + pos, "chunk-signature=", 16)) return MEC_ERR_MALFORMED_ENCODING;
    const uint8_t* claim = b + pos + 16;
    pos += 80;
    for (const uint8_t want : {'\r', '\n'}) {
      if (pos >= blen) return MEC_ERR_INCOMPLETE_BODY;
      if (b[pos++] != want) return MEC_ERR_MALFORMED_ENCODING;
    }
    if (blen - pos < size) return MEC_ERR_INCOMPLETE_BODY;
    o->ch.push_back(AwsChunk{pos, size, o->decoded, prev, claim});
    prev = claim;
    pos += size;
    o->decoded += size;
    if (size == 0) break;
    // the CRLF behind the payload: a missing or cut-off '\r' is malformed, a cut-off '\n' an unexpected EOF
    if (pos >= blen || b[pos] != '\r') return MEC_ERR_MALFORMED_ENCODING;
    if (++pos >= blen) return MEC_ERR_INCOMPLETE_BODY;
    if (b[pos++] != '\n') return MEC_ERR_MALFORMED_ENCODING;
    if (o->decoded > D) return MEC_ERR_OVERREAD;  // the reader yields a chunk only after its signature and CRLF passed
  }
  if (trailer) {
    const int64_t v0 = pos;
    for (;; pos++) {  // the value: every byte up to '\r', which must be followed by '\n'
      if (pos >= blen) return MEC_ERR_INCOMPLETE_BODY;
      if (b[pos] == '\r') break;
    }
    o->tmsg.assign(b + v0, b + pos);
    if (++pos >= blen) return MEC_ERR_INCOMPLETE_BODY;
    if (b[pos++] != '\n') return MEC_ERR_MALFORMED_ENCODING;
    const int64_t s0 = pos;
    for (;; pos++) {  // the signature line up to '\r', then exactly "\n\r\n" (a cut-off part of it is malformed)
      if (pos >= blen) return MEC_ERR_INCOMPLETE_BODY;
      if (b[pos] == '\r') break;
    }
    const int64_t s1 = pos++;
    if (pos >= blen) return MEC_ERR_INCOMPLETE_BODY;
    if (blen - pos < 3 || memcmp(b + pos, "\n\r\n", 3)) return MEC_ERR_MALFORMED_ENCODING;
    static const char kPrefix[] = "x-amz-trailer-signature:";
    const int64_t np = sizeof(kPrefix) - 1;
    if (s1 - s0 < np || memcmp(b + s0, kPrefix, np)) return MEC_ERR_MALFORMED_ENCODING;
    if (!o->tmsg.empty() && o->tmsg.back() != '\n') o->tmsg.push_back('\n');
    const uint8_t* sig = b + s0 + np;
    int64_t sl = s1 - s0 - np;
    trim_space(sig, sl);
    if (sl != 64) return MEC_ERR_SIGNATURE_MISMATCH;
    o->tclaim = sig;
  }
  return o->decoded < D ? MEC_ERR_INCOMPLETE_BODY : MEC_OK;
}

// Per-slot second stream and events of the chunked encode's verify launches, created on first use
static int sig_streams(mec_codec* c) {
  for (auto& s : c->slots) {
    MEC_CUDA_OK(s.st2.create(cudaStreamNonBlocking));
    MEC_CUDA_OK(s.ev_staged.create(cudaEventDisableTiming));
    MEC_CUDA_OK(s.ev_verified.create(cudaEventDisableTiming));
  }
  return MEC_OK;
}

// The aws-chunks of one staging step: [h0, h1) are the rows it verifies, those whose decoded start falls in [own0, own1) (the last
// step: from own0 on, and the trailer row); [a, e) are the chunks it stages, every chunk that overlaps the decoded bytes from `lo`
// on that the step needs, and its rows' chunks.  The steps' [own0, own1) tile the decoded bytes, so every row is verified once;
// the bytes a step needs end at or before own1, so the overlapping chunks end where the rows do.
struct AwsSpan {
  int64_t a, e;    // staged chunks
  int64_t h0, h1;  // verified rows
  bool trow;       // and the trailer row
};
static AwsSpan aws_span(const ChunkedBody& P, int64_t lo, int64_t own0, int64_t own1, bool last) {
  const std::vector<AwsChunk>& ch = P.ch;
  auto first = [&](auto pred) { return std::partition_point(ch.begin(), ch.end(), pred) - ch.begin(); };
  AwsSpan sp;
  const int64_t a1 = first([&](const AwsChunk& x) { return x.doff + x.size <= lo; });  // first chunk that overlaps or follows
  sp.h0 = first([&](const AwsChunk& x) { return x.doff < own0; });
  sp.h1 = last ? static_cast<int64_t>(ch.size()) : first([&](const AwsChunk& x) { return x.doff < own1; });
  sp.a = std::min(a1, sp.h0);
  sp.e = sp.h1;
  sp.trow = last && P.tclaim;
  return sp;
}

// ONE batched copy stages into `buf`, back to back, the payloads of the chunks [sp.a, sp.e), placed so that decoded byte `lo` lands
// 16-byte aligned and the buffer reaches at least decoded byte `hi`; the trailer message follows when the step has the trailer
// row.  *base: decoded byte x is at *base + x.  The step's rows are then verified by ONE launch on the slot's second stream, behind
// the staging, so that the work queued on s.st next does not wait for the hash.  *r0 / *nrow: the first row and the number of rows
// of the step, whose verdicts land behind its rows in s.sig_tab.h once s.st2 has drained.
static int aws_stage(mec_codec* c, Slot& s, DevBuf& buf, const uint8_t* body, const ChunkedBody& P, const AwsSpan& sp, int64_t lo,
                     int64_t hi, uint8_t** base, int64_t* r0, int64_t* nrow) {
  const std::vector<AwsChunk>& ch = P.ch;
  const int64_t a = sp.a, e = sp.e, h0 = sp.h0, h1 = sp.h1;
  const int64_t lo_s = a < e ? ch[a].doff : lo, hi_s = a < e ? ch[e - 1].doff + ch[e - 1].size : lo;
  const int64_t pad = (16 - (lo - lo_s) % 16) % 16;
  const int64_t tpos = round_up(pad + std::max(hi_s, hi) - lo_s, 16);
  int rc;
  if ((rc = buf.ensure(static_cast<size_t>(tpos + (sp.trow ? static_cast<int64_t>(P.tmsg.size()) : 0) + 256)))) return rc;
  uint8_t* b = static_cast<uint8_t*>(buf.p) + pad - lo_s;
  *base = b;
  CopyList list;
  int64_t staged = 0;
  for (int64_t j = a; j < e; j++) {
    list.add(b + ch[j].doff, body + ch[j].pay, ch[j].size);
    staged += ch[j].size;
  }
  if (sp.trow) {
    list.add(static_cast<uint8_t*>(buf.p) + tpos, P.tmsg.data(), static_cast<int64_t>(P.tmsg.size()));
    staged += static_cast<int64_t>(P.tmsg.size());
  }
  if ((rc = list.flush(s.st))) return rc;
  c->st_h2d += staged;
  *r0 = h0;
  *nrow = h1 - h0 + (sp.trow ? 1 : 0);
  if (*nrow == 0) return MEC_OK;
  const size_t tab = static_cast<size_t>(*nrow) * (sizeof(SigRow) + 1);
  if ((rc = s.sig_tab.ensure(tab))) return rc;
  SigRow* h = static_cast<SigRow*>(s.sig_tab.h.p);
  for (int64_t j = h0; j < h1; j++) h[j - h0] = sig_row(b + ch[j].doff, ch[j].size, j - h0, kSigPayload, ch[j].prev, ch[j].claim);
  if (sp.trow)
    h[h1 - h0] = sig_row(static_cast<uint8_t*>(buf.p) + tpos, static_cast<int64_t>(P.tmsg.size()), h1 - h0, kSigTrailer,
                         ch.back().claim, P.tclaim);
  MEC_CUDA_OK(cudaEventRecord(s.ev_staged, s.st));
  MEC_CUDA_OK(cudaStreamWaitEvent(s.st2, s.ev_staged, 0));
  SigRow* d = static_cast<SigRow*>(s.sig_tab.d.p);
  if ((rc = sig_launch(c, h, d, *nrow, s.st2))) return rc;
  MEC_CUDA_OK(cudaMemcpyAsync(h + *nrow, d + *nrow, static_cast<size_t>(*nrow), cudaMemcpyDeviceToHost, s.st2));
  MEC_CUDA_OK(cudaEventRecord(s.ev_verified, s.st2));
  return MEC_OK;
}

// The staging step of mec_encode_chunked for the object bytes [off, off + bytes), `last` for the pipeline's last chunk (or the one
// step of an empty object): the aws-chunks that overlap the range or start in it go to s.src with object byte `off` 16-byte
// aligned for the encode, and the rows of those that start in it are verified.
static int chunked_stage(mec_codec* c, Slot& s, const uint8_t* body, const ChunkedBody& P, int64_t off, int64_t bytes, bool last,
                         Staged* o, int64_t* r0, int64_t* nrow) {
  uint8_t* base;
  const int rc = aws_stage(c, s, s.src, body, P, aws_span(P, off, off, off + bytes, last), off, off + bytes, &base, r0, nrow);
  if (rc) return rc;
  o->obj = o->ck = base + off;
  o->ck_len = bytes;
  return MEC_OK;
}

// The staging step of mec_encode_chunked_sse for the ciphertext bytes [off, off + bytes) of a stream of D plaintext bytes.  The
// packages that overlap the range need the plaintext [pt0, pt1): the aws-chunks that overlap it go to s.aux with pt0 16-byte
// aligned, and the rows whose decoded start falls among the packages that start in the range are verified (the steps' package
// starts tile the plaintext).  The packages are then sealed into s.src as mec_encode_sse seals them.
static int chunked_sse_stage(mec_codec* c, Slot& s, const uint8_t* body, const ChunkedBody& P, int64_t D, int64_t off, int64_t bytes,
                             bool last, Staged* o, int64_t* r0, int64_t* nrow, int chacha) {
  const DareSpan d = dare_span(D, off, bytes);
  const AwsSpan sp = aws_span(P, d.pt0, d.ps * kPkg, (d.p1 + 1) * kPkg, last);
  uint8_t* base;
  const int rc = aws_stage(c, s, s.aux, body, P, sp, d.pt0, d.pt1, &base, r0, nrow);
  if (rc) return rc;
  return dare_seal_chunk(c, s, d, D, base + d.pt0, o, chacha == 2);
}

// newSignV4ChunkedReader + Erasure.Encode (cmd/object-handlers.go:1890, cmd/object-multipart-handlers.go:682,
// cmd/object-handlers.go:2294): the body is de-framed on the host, its payloads go to the device through chunked_stage, and the
// encode runs over the D decoded bytes as mec_encode does.  With an SSE key (mec_encode_chunked_sse: newSignV4ChunkedReader +
// EncryptRequest + Erasure.Encode) the payloads go through chunked_sse_stage instead and the encode runs over their DARE stream as
// mec_encode_sse does.  The caller has checked the arguments.
static int64_t encode_chunked(mec_codec* c, const uint8_t* body, int64_t body_len, int64_t decoded_len, const uint8_t* key,
                              const uint8_t* seed, const char* date, const char* scope, int trailer, const uint8_t* sse_key,
                              const uint8_t* nonce, uint8_t* const* files, int write_quorum, uint8_t* trailer_out, int64_t trailer_cap,
                              int64_t* trailer_len) {
  if (trailer_len) *trailer_len = 0;
  int online = 0;
  for (int i = 0; i < c->n; i++) online += files[i] != nullptr;
  if (online < write_quorum) return MEC_ERR_WRITE_QUORUM;  // cmd/erasure-encode.go:59-65
  ChunkedBody P;
  const int perr = parse_chunked(body, body_len, decoded_len, seed, trailer != 0, &P);
  const int64_t nrows = static_cast<int64_t>(P.ch.size()) + (P.tclaim ? 1 : 0);
  if (nrows == 0) return perr;  // the first header already fails: no signature to check before it
  int rc = require_streaming(c);
  if (rc) return rc;
  if (c->S() >= (1ll << 31)) return MEC_ERR_UNSUPPORTED;
  std::lock_guard<std::mutex> lk(c->mu);
  MEC_CUDA_OK(cudaSetDevice(c->device));
  if ((rc = sig_ensure(c)) || (rc = sig_streams(c))) return rc;
  Slot& s0 = c->slots[0];
  sig_call_host(c, key, date, scope);
  SigScrub scrub{c, s0.st};
  if ((rc = sig_call_upload(c, s0.st))) return rc;
  std::vector<uint8_t> verdict(static_cast<size_t>(nrows), 0);
  int64_t r0[kSlots] = {}, nr[kSlots] = {};
  auto collect = [&](int si) {
    const uint8_t* v = reinterpret_cast<const uint8_t*>(static_cast<const SigRow*>(c->slots[si].sig_tab.h.p) + nr[si]);
    memcpy(verdict.data() + r0[si], v, static_cast<size_t>(nr[si]));
  };
  const int64_t D = decoded_len;
  const int64_t len = sse_key ? mec_dare_encrypted_size(D) : D;  // the bytes the encode covers
  const int chacha = c->dare_chacha20.load();
  if (D == 0) {  // no encode: the rows of the empty object in one step
    Staged sg;
    if ((rc = chunked_stage(c, s0, body, P, 0, 0, true, &sg, &r0[0], &nr[0]))) return rc;
    MEC_CUDA_OK(cudaStreamSynchronize(s0.st2));
    collect(0);
  } else {
    auto run = [&]() -> int {
      return encode_pipeline(
          c, len,
          [&](Slot& s, int64_t off, int64_t bytes, Staged* o) -> int {
            const int si = static_cast<int>(&s - c->slots);
            const bool last = off + bytes == len;
            if (sse_key) return chunked_sse_stage(c, s, body, P, D, off, bytes, last, o, &r0[si], &nr[si], chacha);
            return chunked_stage(c, s, body, P, off, bytes, last, o, &r0[si], &nr[si]);
          },
          [&](const EncChunk& ch) -> int {
            const int e = frames_enqueue_chunk(c, ch, files, true, nullptr);
            if (e) return e;
            if (nr[ch.s - c->slots]) MEC_CUDA_OK(cudaStreamWaitEvent(ch.st, ch.s->ev_verified, 0));  // the slot drains its verify too
            return MEC_OK;
          },
          [&](const EncChunk& ch) {
            frames_retire(c, ch, files, true, nullptr);
            collect(static_cast<int>(ch.s - c->slots));
          });
    };
    if (sse_key) {
      if ((rc = dare_keys(c, 1, sse_key, nonce, s0.st, chacha))) return rc;
      DareScrub dscrub{c, 1, s0.st};
      MEC_CUDA_OK(cudaStreamSynchronize(s0.st));  // every slot stream reads the keys
      rc = run();
    } else {
      rc = run();
    }
    if (rc) return rc;
  }
  for (uint8_t v : verdict)
    if (!v) return MEC_ERR_SIGNATURE_MISMATCH;  // every row precedes the point where the serial reader stopped
  if (perr) return perr;
  if (D == 0 && c->checksums) {  // the empty stream's checksums, as reset_last_checksums leaves them
    for (auto& v : c->last_crc) v = 0;
    c->last_crc_len = 0;
  }
  if (trailer) {
    *trailer_len = static_cast<int64_t>(P.tmsg.size());
    if (trailer_cap > 0) memcpy(trailer_out, P.tmsg.data(), static_cast<size_t>(std::min<int64_t>(trailer_cap, *trailer_len)));
  }
  return D;
}

// mec_encode_chunked's argument checks
static bool chunked_args_ok(const mec_codec* c, const uint8_t* body, int64_t body_len, int64_t decoded_len, const uint8_t* key,
                            const uint8_t* seed, const char* date, const char* scope, int trailer, uint8_t* const* files,
                            const uint8_t* trailer_out, int64_t trailer_cap, const int64_t* trailer_len) {
  if (!c || body_len < 0 || (body_len > 0 && !body) || decoded_len < 0 || !key || !seed || !date || !scope || !files) return false;
  if (trailer && (!trailer_len || trailer_cap < 0 || (trailer_cap > 0 && !trailer_out))) return false;
  return lower_hex64(seed) && strlen(date) + strlen(scope) + 2 <= static_cast<size_t>(kSigMaxHead);
}

extern "C" int64_t mec_encode_chunked(mec_codec* c, const uint8_t* body, int64_t body_len, int64_t decoded_len, const uint8_t* key,
                                      const uint8_t* seed, const char* date, const char* scope, int trailer, uint8_t* const* files,
                                      int write_quorum, uint8_t* trailer_out, int64_t trailer_cap, int64_t* trailer_len) {
  NvtxRange nvtx("mec_encode_chunked");
  if (!chunked_args_ok(c, body, body_len, decoded_len, key, seed, date, scope, trailer, files, trailer_out, trailer_cap, trailer_len))
    return MEC_ERR_INVALID_ARGUMENT;
  return encode_chunked(c, body, body_len, decoded_len, key, seed, date, scope, trailer, nullptr, nullptr, files, write_quorum,
                        trailer_out, trailer_cap, trailer_len);
}

// newSignV4ChunkedReader + EncryptRequest + Erasure.Encode (cmd/object-handlers.go:1892, :2070): mec_encode_chunked's de-framing and
// verdicts, and mec_encode_sse's part files of the decoded bytes, in one pass of the encode pipeline.
extern "C" int64_t mec_encode_chunked_sse(mec_codec* c, const uint8_t* body, int64_t body_len, int64_t decoded_len,
                                          const uint8_t* sig_key, const uint8_t* seed, const char* date, const char* scope, int trailer,
                                          const uint8_t* sse_key, const uint8_t* nonce, uint8_t* const* files, int write_quorum,
                                          uint8_t* trailer_out, int64_t trailer_cap, int64_t* trailer_len) {
  NvtxRange nvtx("mec_encode_chunked_sse");
  if (!chunked_args_ok(c, body, body_len, decoded_len, sig_key, seed, date, scope, trailer, files, trailer_out, trailer_cap, trailer_len) ||
      !sse_key || !nonce)
    return MEC_ERR_INVALID_ARGUMENT;
  const int64_t E = mec_dare_encrypted_size(decoded_len);
  if (E < 0) return E;
  return encode_chunked(c, body, body_len, decoded_len, sig_key, seed, date, scope, trailer, sse_key, nonce, files, write_quorum,
                        trailer_out, trailer_cap, trailer_len);
}

// Batched heal (SURVEY §8f rank 2, BASELINE config 4): objects are independent, so a pool of codec handles — each with
// its own streams and staging buffers — is driven by one host thread per handle; the H2D staging of one object then
// overlaps the kernel and the D2H of the others (healObject's callers, cmd/global-heal.go:152, do the same with goroutines).
// rcs[o] = MEC_ERR_FILE_CORRUPT means "healed, but a source reader of object o failed its digest" (see mec_heal_prefer);
// the return value is the first result that is neither MEC_OK nor that.
extern "C" int mec_heal_batch(mec_codec* const* pool, int npool, int64_t nobjects, const uint8_t* const* const* files,
                              const int64_t* totals, uint8_t* const* const* out_files, int* rcs) {
  if (!pool || npool <= 0 || nobjects < 0 || (nobjects > 0 && (!files || !totals || !out_files))) return MEC_ERR_INVALID_ARGUMENT;
  for (int i = 0; i < npool; i++)
    if (!pool[i]) return MEC_ERR_INVALID_ARGUMENT;
  std::atomic<int64_t> next{0};
  std::atomic<int> first_err{MEC_OK};
  auto work = [&](int w) {
    for (;;) {
      const int64_t o = next.fetch_add(1);
      if (o >= nobjects) return;
      const int rc = mec_heal(pool[w], files[o], totals[o], out_files[o]);
      if (rcs) rcs[o] = rc;
      if (rc != MEC_OK && rc != MEC_ERR_FILE_CORRUPT) {
        int expected = MEC_OK;
        first_err.compare_exchange_strong(expected, rc);
      }
    }
  };
  const int nthreads = static_cast<int>(std::min<int64_t>(npool, nobjects));
  std::vector<std::thread> th;
  for (int w = 1; w < nthreads; w++) th.emplace_back(work, w);
  if (nthreads > 0) work(0);
  for (auto& t : th) t.join();
  return first_err.load();
}

// The hash-only check (k = 1, r = 0) of `nframes` frames staged in slot `s` at `base` (frame j at base + j*P: its 32-byte digest, then
// lens[j] shard bytes; (arena_frames - j) * P + 512 readable bytes from frame j on), enqueued on the slot's stream.  `lens` is
// page-locked host memory.  one_launch (the codec's options allow the latency kernel at this size): every frame, full or short,
// hashes in ONE launch with a per-frame length table.  Otherwise one launch over each run of full frames and one per short frame
// (a short frame's digest covers fewer bytes).  Verdicts come back to s.flags.h[0, nframes).  Shared by bitrotVerify on a codec
// (verify_files_locked) and merged verify batches (batcher_submit_verify).
static int verify_frames(mec_codec* c, Slot& s, const uint8_t* base, int64_t arena_frames, int64_t nframes, const int32_t* lens, bool one_launch) {
  const int64_t S = c->S(), P = round_up(32 + S, 16);
  int rc;
  if ((rc = s.dig.d.ensure(static_cast<size_t>(nframes * 32)))) return rc;
  if ((rc = s.flags.ensure(static_cast<size_t>(nframes)))) return rc;
  MEC_CUDA_OK(cudaMemsetAsync(s.flags.d.p, 0, static_cast<size_t>(nframes), s.st));
  const int32_t* block_len = nullptr;
  auto launch = [&](int64_t slot0, int64_t cnt, int64_t len) -> int {
    FusedDesc d;
    d.k = 1; d.r = 0; d.contiguous = false; d.key = kMagicKey;
    d.block_len = block_len;
    d.in_block_stride = P; d.expect_block_stride = P;
    const uint8_t* at = base + slot0 * P;
    d.nblocks = cnt; d.S = static_cast<int32_t>(len);
    d.map_base[0] = at; d.map_len[0] = (arena_frames - slot0) * P + 512;
    d.expect_ptr[0] = at; d.in_ptr[0] = at + 32;
    d.digests = static_cast<uint8_t*>(s.dig.d.p) + slot0 * 32;
    d.corrupt = static_cast<uint8_t*>(s.flags.d.p) + slot0;
    return c->eng->launch_fused(d, c->opt, s.st);
  };
  if (one_launch) {
    if ((rc = s.dreq.d.ensure(static_cast<size_t>(nframes) * sizeof(int32_t)))) return rc;
    MEC_CUDA_OK(cudaMemcpyAsync(s.dreq.d.p, lens, static_cast<size_t>(nframes) * sizeof(int32_t), cudaMemcpyHostToDevice, s.st));
    block_len = static_cast<const int32_t*>(s.dreq.d.p);
    if ((rc = launch(0, nframes, S))) return rc;
  } else {
    // runs of full frames between the short ones
    int64_t at = 0;
    for (int64_t j = 0; j <= nframes; j++) {
      if (j < nframes && lens[j] == S) continue;
      if (j > at && (rc = launch(at, j - at, S))) return rc;
      if (j < nframes && (rc = launch(j, 1, lens[j]))) return rc;
      at = j + 1;
    }
  }
  MEC_CUDA_OK(s.flags.download(static_cast<size_t>(nframes), s.st));
  c->st_blocks_read += nframes;
  return MEC_OK;
}

static inline bool is_whole_algo(int a) { return a == MEC_SHA256 || a == MEC_HIGHWAYHASH256 || a == MEC_BLAKE2B512; }

// bitrotVerify (cmd/bitrot.go:164-215), streaming algorithm: every frame's digest is recomputed and compared.  The scan of one
// or many shard files (the scanner's deep-scan visits every part of every drive of an object: cmd/xl-storage.go:2550-2600) is cut
// into chunks of frames that run through the codec's slots: staging of chunk c+1 overlaps the hash-only launch of chunk c
// (verify_frames); a chunk's verdicts come back when its slot is reused.  Files with results[f] != MEC_OK, an empty part or (with
// `algos`) a whole-file algorithm are skipped; result[f] = MEC_ERR_FILE_CORRUPT where a frame fails.
static int verify_files_locked(mec_codec* c, int64_t nfiles, const uint8_t* const* files, const int64_t* part_lens, const int* algos,
                               int* results) {
  const int64_t S = c->S(), fstride = 32 + S, P = round_up(32 + S, 16);
  MEC_CUDA_OK(cudaSetDevice(c->device));
  SlotDrain drain(c);
  struct Piece { int64_t file, nb; };
  std::vector<Piece> inflight[kSlots];
  const int64_t chunk = std::max<int64_t>(1, (32ll << 20) / fstride);  // frames per chunk (~32 MiB)
  int rc;
  SlotRing ring(c, [&](int si) {
    const uint8_t* fl = static_cast<const uint8_t*>(c->slots[si].flags.h.p);
    int64_t o = 0;
    for (const Piece& pc : inflight[si]) {
      for (int64_t b = 0; b < pc.nb; b++)
        if (fl[o + b]) results[pc.file] = MEC_ERR_FILE_CORRUPT;
      o += pc.nb;
    }
    inflight[si].clear();
  });
  int64_t f = 0, b0 = 0;  // next file / next frame of it
  while (f < nfiles) {
    if ((rc = ring.acquire())) return rc;
    const int si = ring.si;
    Slot& s = c->slots[si];
    if ((rc = s.src.ensure(static_cast<size_t>(chunk * P + 512)))) return rc;
    if ((rc = s.dreq.h.ensure(static_cast<size_t>(chunk) * sizeof(int32_t)))) return rc;
    int64_t used = 0;
    // fill the chunk with frames of consecutive files.  When the chunk is a launch the latency kernel takes (it is, unless options
    // say otherwise: ~380 frames of a 1 MiB-block part file), short runs of frames are staged by ONE batched copy call: a scan over
    // thousands of small part files costs two driver calls per 32 MiB, not two per file.
    const bool one_launch = c->eng->small_ok(c->opt, chunk);
    CopyList list;
    int32_t* lens = static_cast<int32_t*>(s.dreq.h.p);
    while (f < nfiles && used < chunk) {
      if (results[f] != MEC_OK || part_lens[f] == 0 || (algos && algos[f] != MEC_HIGHWAYHASH256S)) { f++; b0 = 0; continue; }
      const int64_t nblocks = ceil_frac(part_lens[f], S), last_len = part_lens[f] - (nblocks - 1) * S;
      const int64_t take = std::min(chunk - used, nblocks - b0);
      FrameGeom sub{take, S, (b0 + take == nblocks) ? last_len : S};
      for (int64_t j = 0; j < take; j++) lens[used + j] = static_cast<int32_t>((j == take - 1) ? sub.last_len : S);
      if (one_launch && take < kBatchedCopyBlocks) {
        for (int64_t j = 0; j < take; j++)
          list.add(static_cast<uint8_t*>(s.src.p) + (used + j) * P, files[f] + (b0 + j) * fstride, 32 + lens[used + j]);
      } else if ((rc = stage_frames(files[f] + b0 * fstride, static_cast<uint8_t*>(s.src.p) + used * P, sub, s.st))) return rc;
      c->st_h2d += sub.file_bytes();
      inflight[si].push_back(Piece{f, take});
      used += take;
      b0 += take;
      if (b0 == nblocks) { f++; b0 = 0; }
    }
    if (used == 0) break;
    if ((rc = list.flush(s.st))) return rc;
    if ((rc = verify_frames(c, s, static_cast<const uint8_t*>(s.src.p), chunk, used, lens, one_launch))) return rc;
    ring.submitted();
  }
  return ring.finish();
}

// Legacy parts of a verify call (mec_bitrot_verify_parts): every part p with results[p] == MEC_OK and a whole-file algorithm is
// hashed whole and compared with the first mec_digest_size bytes of sums + p*64 (cmd/bitrot.go:165-174).  Parts are staged in
// input order in groups of at most kVerifyWholeGroupBytes file bytes (a larger file alone), each group by ONE batched copy into
// slot 0 and ONE whole_hash_kernel launch whose algorithm groups hold its SHA256, HighwayHash256 and BLAKE2b512 parts.
constexpr int64_t kVerifyWholeGroupBytes = 256ll << 20;
static const int kWholeAlgos[kWholeGroups] = {MEC_SHA256, MEC_HIGHWAYHASH256, MEC_BLAKE2B512};
static inline int whole_group(int algo) { return algo == MEC_SHA256 ? 0 : algo == MEC_HIGHWAYHASH256 ? 1 : 2; }

static int whole_hash_groups(mec_codec* c, int ngroups, const int* algos, const int64_t* counts, const uint8_t* d_data, int64_t pitch,
                             int64_t len, uint8_t* d_out, cudaStream_t st, const WholeStream* streams);
static int verify_whole_locked(mec_codec* c, int64_t nparts, const int* algos, const uint8_t* const* files, const int64_t* file_lens,
                               const uint8_t* sums, int* results) {
  MEC_CUDA_OK(cudaSetDevice(c->device));
  Slot& s = c->slots[0];
  SlotDrain drain(s);
  int rc;
  int64_t p = 0;
  std::vector<int64_t> group[kWholeGroups];
  while (p < nparts) {
    for (auto& g : group) g.clear();
    int64_t bytes = 0, nfiles = 0;
    for (; p < nparts; p++) {
      if (results[p] != MEC_OK || !is_whole_algo(algos[p])) continue;
      if (nfiles > 0 && bytes + file_lens[p] > kVerifyWholeGroupBytes) break;
      group[whole_group(algos[p])].push_back(p);
      bytes += file_lens[p];
      nfiles++;
    }
    if (nfiles == 0) break;
    // the file arena as batch_whole_stage lays it out: each file 16-byte aligned with 256 readable bytes behind it
    const size_t tab_bytes = static_cast<size_t>(nfiles) * sizeof(WholeStream);
    if ((rc = s.wtab.ensure(tab_bytes))) return rc;
    if ((rc = s.wdig.ensure(static_cast<size_t>(nfiles) * 64))) return rc;
    WholeStream* ws = static_cast<WholeStream*>(s.wtab.h.p);
    int64_t arena = 0, j = 0, counts[kWholeGroups];
    for (int g = 0; g < kWholeGroups; g++) {
      counts[g] = static_cast<int64_t>(group[g].size());
      for (int64_t q : group[g]) {
        ws[j++] = WholeStream{arena, file_lens[q]};
        arena += round_up(file_lens[q], 16) + 256;
      }
    }
    if ((rc = s.src.ensure(static_cast<size_t>(arena)))) return rc;
    uint8_t* d = static_cast<uint8_t*>(s.src.p);
    MEC_CUDA_OK(s.wtab.upload(tab_bytes, s.st));
    CopyList list;
    j = 0;
    for (int g = 0; g < kWholeGroups; g++)
      for (int64_t q : group[g]) list.add(d + ws[j++].off, files[q], file_lens[q]);
    if ((rc = list.flush(s.st))) return rc;
    if ((rc = whole_hash_groups(c, kWholeGroups, kWholeAlgos, counts, d, 0, 0, static_cast<uint8_t*>(s.wdig.d.p), s.st,
                                static_cast<const WholeStream*>(s.wtab.d.p))))
      return rc;
    c->eng->count_launch();
    MEC_CUDA_OK(s.wdig.download(static_cast<size_t>(nfiles) * 64, s.st));
    MEC_CUDA_OK(cudaStreamSynchronize(s.st));
    c->st_h2d += bytes;
    const uint8_t* got = static_cast<const uint8_t*>(s.wdig.h.p);
    j = 0;
    for (int g = 0; g < kWholeGroups; g++)
      for (int64_t q : group[g])
        if (memcmp(got + 64 * j++, sums + q * 64, static_cast<size_t>(mec_digest_size(algos[q]))))
          results[q] = MEC_ERR_FILE_CORRUPT;  // cmd/bitrot.go:171-173
  }
  return MEC_OK;
}

// The decisions of a verify call that need no device (mec_bitrot_verify_parts' per-part refusals, bitrotVerify's length check);
// parts left at MEC_OK with bytes to hash are counted in *frames (streaming frames) and *whole (whole-file parts).
static void verify_decide(int64_t S, int64_t nparts, const int* algos, const uint8_t* const* files, const int64_t* file_lens,
                          const int64_t* part_lens, int* results, int64_t* frames, int64_t* whole) {
  *frames = *whole = 0;
  for (int64_t p = 0; p < nparts; p++) {
    const int a = algos[p];
    const bool streaming = a == MEC_HIGHWAYHASH256S;
    int r = MEC_OK;
    if ((!streaming && !is_whole_algo(a)) || file_lens[p] < 0 || (streaming && part_lens[p] < 0) || (!files[p] && file_lens[p] > 0))
      r = MEC_ERR_INVALID_ARGUMENT;
    else if (streaming && file_lens[p] != mec_bitrot_shard_file_size(part_lens[p], S, a))
      r = MEC_ERR_FILE_CORRUPT;  // cmd/bitrot.go:183
    else if (streaming)
      *frames += ceil_frac(part_lens[p], S);
    else
      (*whole)++;
    results[p] = r;
  }
}

// mec_bitrot_verify_parts' refusals before any device work
static bool verify_args_ok(int64_t nparts, const int* algos, const uint8_t* const* files, const int64_t* file_lens, const int64_t* part_lens,
                           const uint8_t* sums, const int* results) {
  if (nparts < 0 || (nparts > 0 && (!algos || !files || !file_lens || !part_lens || !results))) return false;
  if (!sums)
    for (int64_t p = 0; p < nparts; p++)
      if (is_whole_algo(algos[p])) return false;
  return true;
}

// Device work of a verify call whose per-part decisions are made (results[p] == MEC_OK: hash it), on the locked codec
static int verify_parts_locked(mec_codec* c, int64_t nparts, const int* algos, const uint8_t* const* files, const int64_t* file_lens,
                               const int64_t* part_lens, const uint8_t* sums, int* results, int64_t frames, int64_t whole) {
  int rc;
  if ((rc = ensure_engine(c))) return rc;
  if (frames > 0 && (rc = verify_files_locked(c, nparts, files, part_lens, algos, results))) return rc;
  if (whole > 0 && (rc = verify_whole_locked(c, nparts, algos, files, file_lens, sums, results))) return rc;
  return MEC_OK;
}

extern "C" int mec_bitrot_verify_parts(mec_codec* c, int64_t nparts, const int* algos, const uint8_t* const* files, const int64_t* file_lens,
                                       const int64_t* part_lens, const uint8_t* sums, int* results) {
  NvtxRange nvtx("mec_bitrot_verify_parts");
  if (!c || !verify_args_ok(nparts, algos, files, file_lens, part_lens, sums, results)) return MEC_ERR_INVALID_ARGUMENT;
  int64_t frames = 0, whole = 0;
  verify_decide(c->S(), nparts, algos, files, file_lens, part_lens, results, &frames, &whole);
  if (frames == 0 && whole == 0) return MEC_OK;
  std::lock_guard<std::mutex> lk(c->mu);
  return verify_parts_locked(c, nparts, algos, files, file_lens, part_lens, sums, results, frames, whole);
}

// bitrotVerify of streaming part files on a HighwayHash256S codec: mec_bitrot_verify_parts with every part HighwayHash256S, and the
// call's own argument rules (a NULL file with a non-empty part is refused per file)
extern "C" int mec_bitrot_verify_batch(mec_codec* c, int64_t nfiles, const uint8_t* const* files, const int64_t* file_lens,
                                       const int64_t* part_lens, int* results) {
  if (!c || nfiles < 0 || (nfiles > 0 && (!files || !file_lens || !part_lens || !results))) return MEC_ERR_INVALID_ARGUMENT;
  const int64_t S = c->S();
  int64_t frames = 0;
  for (int64_t f = 0; f < nfiles; f++) {
    results[f] = MEC_OK;
    if (!files[f] && part_lens[f] > 0) { results[f] = MEC_ERR_INVALID_ARGUMENT; continue; }
    if (file_lens[f] != mec_bitrot_shard_file_size(part_lens[f], S, c->algo)) results[f] = MEC_ERR_FILE_CORRUPT;  // cmd/bitrot.go:183
    else if (part_lens[f] > 0) frames += ceil_frac(part_lens[f], S);
  }
  if (frames == 0) return MEC_OK;
  int rc = require_streaming(c);
  if (rc) return rc;
  std::lock_guard<std::mutex> lk(c->mu);
  return verify_parts_locked(c, nfiles, nullptr, files, file_lens, part_lens, nullptr, results, frames, 0);
}

extern "C" int mec_bitrot_verify(mec_codec* c, const uint8_t* file, int64_t file_len, int64_t part_len) {
  if (!c || !file) return MEC_ERR_INVALID_ARGUMENT;
  int result = MEC_OK;
  const int rc = mec_bitrot_verify_batch(c, 1, &file, &file_len, &part_len, &result);
  return rc ? rc : result;
}

// ------------------------------------------------------------------------------------------------
// legacy whole-file bitrot algorithms
extern "C" int mec_digest_size(int algo) {
  switch (algo) {
    case MEC_SHA256: case MEC_HIGHWAYHASH256: case MEC_HIGHWAYHASH256S: return 32;
    case MEC_BLAKE2B512: return 64;
  }
  return -1;
}

// ONE whole_hash_kernel launch over `ngroups` algorithm groups: group g is the next counts[g] streams, of algorithm algos[g], at
// d_data + s*pitch of `len` bytes each or, with a device stream table, at d_data + streams[s].off of streams[s].len bytes.  Each
// group starts on a warp boundary.  Empty groups are dropped.
static int whole_hash_groups(mec_codec* c, int ngroups, const int* algos, const int64_t* counts, const uint8_t* d_data, int64_t pitch,
                             int64_t len, uint8_t* d_out, cudaStream_t st, const WholeStream* streams) {
  WholeHashParams hp;
  memset(&hp, 0, sizeof(hp));
  hp.data = d_data; hp.pitch = pitch; hp.len = len; hp.streams = streams; hp.out = d_out;
  memcpy(hp.key, kMagicKey, 32);
  int64_t stream = 0, thread = 0;
  for (int g = 0; g < ngroups; g++) {
    if (counts[g] == 0) continue;
    const int a = algos[g] == MEC_HIGHWAYHASH256S ? MEC_HIGHWAYHASH256 : algos[g];
    const int q = hp.ngroups++;
    thread = round_up(thread, 32);
    hp.galgo[q] = a; hp.gstream[q] = static_cast<int>(stream); hp.gthread[q] = static_cast<int>(thread);
    stream += counts[g];
    thread += (a == MEC_HIGHWAYHASH256 ? 2 : 1) * counts[g];
  }
  hp.gstream[hp.ngroups] = static_cast<int>(stream);
  if (hp.ngroups == 0) return MEC_OK;
  const int threads = 64;
  whole_hash_kernel<<<static_cast<unsigned>((thread + threads - 1) / threads), threads, 0, st>>>(hp);
  MEC_CUDA_OK(cudaGetLastError());
  c->st_whole_hash++;
  return MEC_OK;
}
// `count` streams of one algorithm (whole_hash_groups with one group)
static int whole_hash_device(mec_codec* c, int algo, const uint8_t* d_data, int64_t pitch, int64_t len, int64_t count,
                             uint8_t* d_out, cudaStream_t st, const WholeStream* streams = nullptr) {
  return whole_hash_groups(c, 1, &algo, &count, d_data, pitch, len, d_out, st, streams);
}

extern "C" int mec_whole_hash(mec_codec* c, int algo, const uint8_t* msgs, int64_t msg_len, int64_t count, uint8_t* digests) {
  if (!c || msg_len < 0 || count < 0 || mec_digest_size(algo) < 0) return MEC_ERR_INVALID_ARGUMENT;
  if (count == 0) return MEC_OK;
  if (count >= (1ll << 30)) return MEC_ERR_UNSUPPORTED;
  std::lock_guard<std::mutex> lk(c->mu);
  int rc;
  if ((rc = ensure_engine(c))) return rc;
  MEC_CUDA_OK(cudaSetDevice(c->device));
  Slot& s = c->slots[0];
  const int64_t pitch = round_up(msg_len, 16) + 128;  // the kernel reads whole 16-byte vectors
  if ((rc = s.src.ensure(static_cast<size_t>(count * pitch + 256)))) return rc;
  if ((rc = s.dig.d.ensure(static_cast<size_t>(count * 64)))) return rc;
  if (msg_len > 0)
    MEC_CUDA_OK(cudaMemcpy2DAsync(s.src.p, static_cast<size_t>(pitch), msgs, static_cast<size_t>(msg_len), static_cast<size_t>(msg_len),
                                  static_cast<size_t>(count), cudaMemcpyHostToDevice, s.st));
  if ((rc = whole_hash_device(c, algo, static_cast<const uint8_t*>(s.src.p), pitch, msg_len, count, static_cast<uint8_t*>(s.dig.d.p), s.st))) return rc;
  const int ds = mec_digest_size(algo);
  MEC_CUDA_OK(cudaMemcpy2DAsync(digests, static_cast<size_t>(ds), s.dig.d.p, 64, static_cast<size_t>(ds), static_cast<size_t>(count),
                                cudaMemcpyDeviceToHost, s.st));
  MEC_CUDA_OK(cudaStreamSynchronize(s.st));
  c->eng->count_launch();
  return MEC_OK;
}

extern "C" int mec_whole_hash_device(mec_codec* c, int algo, const uint8_t* d_msgs, int64_t pitch, int64_t msg_len, int64_t count,
                                     uint8_t* d_digests, void* stream) {
  if (!c || msg_len < 0 || count < 0 || mec_digest_size(algo) < 0 || (pitch & 15) || pitch < msg_len) return MEC_ERR_INVALID_ARGUMENT;
  // the kernel reads every message with 16-byte vector loads and HighwayHash stores its digests as 64-bit words
  if ((msg_len > 0 && count > 0 && !d_msgs) || (reinterpret_cast<uintptr_t>(d_msgs) & 15) || !d_digests ||
      (reinterpret_cast<uintptr_t>(d_digests) & 7))
    return MEC_ERR_INVALID_ARGUMENT;
  if (count == 0) return MEC_OK;
  if (count >= (1ll << 30)) return MEC_ERR_UNSUPPORTED;
  std::lock_guard<std::mutex> lk(c->mu);
  int rc;
  if ((rc = ensure_engine(c))) return rc;
  MEC_CUDA_OK(cudaSetDevice(c->device));
  if ((rc = whole_hash_device(c, algo, d_msgs, pitch, msg_len, count, d_digests, static_cast<cudaStream_t>(stream)))) return rc;
  c->eng->count_launch();
  return MEC_OK;
}

extern "C" int mec_bitrot_verify_whole(mec_codec* c, int algo, const uint8_t* file, int64_t file_len, const uint8_t* want) {
  if (!c || !want || file_len < 0) return MEC_ERR_INVALID_ARGUMENT;
  uint8_t got[64];
  int rc = mec_whole_hash(c, algo, file, file_len, 1, got);
  if (rc) return rc;
  return memcmp(got, want, static_cast<size_t>(mec_digest_size(algo))) ? MEC_ERR_FILE_CORRUPT : MEC_OK;  // cmd/bitrot.go:171-173
}

extern "C" int64_t mec_encode_whole(mec_codec* c, const uint8_t* src, int64_t len, uint8_t* const* files, uint8_t* sums,
                                    int write_quorum) {
  if (!c || len < 0 || !files) return MEC_ERR_INVALID_ARGUMENT;
  if (c->algo == MEC_HIGHWAYHASH256S) return MEC_ERR_INVALID_ARGUMENT;
  int online = 0;
  for (int i = 0; i < c->n; i++) online += files[i] != nullptr;
  if (online < write_quorum) return MEC_ERR_WRITE_QUORUM;
  if (c->S() >= (1ll << 31)) return MEC_ERR_UNSUPPORTED;
  std::lock_guard<std::mutex> lk(c->mu);
  int rc;
  if ((rc = ensure_engine(c))) return rc;
  MEC_CUDA_OK(cudaSetDevice(c->device));
  const int k = c->k, m = c->m, n = c->n;
  const int64_t bs = c->block_size, S = c->S(), pitch = round_up(S, 16);
  const int64_t nall = ceil_frac(len, bs), flen = mec_shard_file_size(c, len), fpitch = round_up(flen, 16) + 128;
  Slot& s = c->slots[0];
  if ((rc = s.src.ensure(static_cast<size_t>(round_up(len, 16) + 256)))) return rc;
  if ((rc = s.out.ensure(static_cast<size_t>(std::max<int64_t>(nall, 1) * std::max(m, 1) * pitch)))) return rc;
  if ((rc = s.aux.ensure(static_cast<size_t>(n * fpitch + 256)))) return rc;
  if ((rc = s.dig.d.ensure(static_cast<size_t>(n * 64)))) return rc;
  if (len > 0) {
    MEC_CUDA_OK(cudaMemcpyAsync(s.src.p, src, static_cast<size_t>(len), cudaMemcpyHostToDevice, s.st));
    if (m > 0) {  // parity only: the hash is not per block for these algorithms
      const int64_t nfull = len / bs, tail = len % bs;
      FusedDesc d;
      d.k = k; d.r = m; d.coef = c->matrix.data() + static_cast<size_t>(k) * k; d.static_encode = true; d.contiguous = true;
      d.key = kMagicKey; d.out_pitch = pitch; d.digests = nullptr;
      if (nfull > 0) {
        d.nblocks = nfull; d.S = static_cast<int32_t>(S); d.in_base = static_cast<const uint8_t*>(s.src.p);
        d.in_block_stride = bs; d.in_block_len = bs; d.out = static_cast<uint8_t*>(s.out.p);
        if ((rc = c->eng->launch_fused(d, c->opt, s.st))) return rc;
      }
      if (tail > 0) {
        d.nblocks = 1; d.S = static_cast<int32_t>(ceil_frac(tail, k)); d.in_base = static_cast<const uint8_t*>(s.src.p) + nfull * bs;
        d.in_block_stride = round_up(tail, 16); d.in_block_len = tail; d.out = static_cast<uint8_t*>(s.out.p) + nfull * m * pitch;
        if ((rc = c->eng->launch_fused(d, c->opt, s.st))) return rc;
      }
    }
    GatherParams gp;
    gp.src = static_cast<const uint8_t*>(s.src.p); gp.parity = static_cast<const uint8_t*>(s.out.p); gp.parity_pitch = pitch;
    gp.block_size = bs; gp.len = len; gp.k = k; gp.m = m; gp.S = S; gp.files = static_cast<uint8_t*>(s.aux.p);
    gp.file_pitch = fpitch; gp.file_len = flen;
    const unsigned gx = static_cast<unsigned>(std::min<int64_t>((flen + 255) / 256, 4096));
    gather_shard_files_kernel<<<dim3(gx, static_cast<unsigned>(n)), 256, 0, s.st>>>(gp);
    MEC_CUDA_OK(cudaGetLastError());
    c->eng->count_launch();
  }
  if ((rc = whole_hash_device(c, c->algo, static_cast<const uint8_t*>(s.aux.p), fpitch, flen, n, static_cast<uint8_t*>(s.dig.d.p), s.st))) return rc;
  c->eng->count_launch();
  for (int i = 0; i < n; i++)
    if (files[i] && flen > 0)
      MEC_CUDA_OK(cudaMemcpyAsync(files[i], static_cast<uint8_t*>(s.aux.p) + i * fpitch, static_cast<size_t>(flen), cudaMemcpyDeviceToHost, s.st));
  if (sums) MEC_CUDA_OK(cudaMemcpyAsync(sums, s.dig.d.p, static_cast<size_t>(n * 64), cudaMemcpyDeviceToHost, s.st));
  MEC_CUDA_OK(cudaStreamSynchronize(s.st));
  return len;
}

// ------------------------------------------------------------------------------------------------
// Decode / Heal over whole-file bitrot readers (cmd/bitrot-whole.go:66-81): a wholeBitrotReader reads its shard file on the first
// ReadAt and checks the digest of the WHOLE file (xlStorage.ReadFile with a verifier, cmd/xl-storage.go:1931-1950) — a mismatch
// is errFileCorrupt, the reader is dropped and parallelReader moves on to the next drive.  Here: the first k readers in index
// order are staged and hashed on the GPU (whole_hash_kernel), failing ones are replaced by the next alive reader until k
// verified shard files sit on the device; the rebuild then runs on those raw shards (no per-block digests exist in this format).
static int require_whole(mec_codec* c) {
  if (c->algo == MEC_HIGHWAYHASH256S) {
    set_last_error("whole-file entry points need a codec created with SHA256, BLAKE2b512 or HighwayHash256");
    return MEC_ERR_INVALID_ARGUMENT;
  }
  return ensure_engine(c);
}

// stage + verify: on return chosen[0..k) (ascending) name k verified files, file chosen[t] at s.aux + pos[t]*fpitch.  Readers are
// taken as parallelReader takes them (`prefer` first, see choose_readers), in rounds of whole_round until k have verified.
static int stage_verified_whole(mec_codec* c, const uint8_t* const* files, const uint8_t* sums, int64_t sfs, uint8_t* alive,
                                uint8_t* corrupt, int* chosen, int* pos, int64_t fpitch, Slot& s, const uint8_t* prefer = nullptr,
                                bool one_launch = false) {
  const int k = c->k, n = c->n;
  int rc;
  if ((rc = s.aux.ensure(static_cast<size_t>(k * fpitch + 256)))) return rc;
  if ((rc = s.dig.ensure(static_cast<size_t>(k * 64)))) return rc;
  WholeSet w{files, sums, nullptr, c->algo, sfs, fpitch, static_cast<uint8_t*>(s.aux.p), static_cast<uint8_t*>(s.dig.d.p),
             static_cast<uint8_t*>(s.dig.h.p), {}};
  for (int i = 0; i < n; i++) w.slot_of[i] = -1;
  for (bool dropped = true; dropped;) {
    int want[kMaxShards];
    if (choose_readers(c, files, alive, prefer, want) < k) return MEC_ERR_READ_QUORUM;
    if ((rc = whole_round(c, w, want, k, alive, corrupt, one_launch, s.st, &dropped))) return rc;
  }
  // compact into ascending order: position t must hold the t-th chosen file (decode rows are defined on ascending indices)
  int nch = 0;
  for (int i = 0; i < n && nch < k; i++)
    if (alive[i] && w.slot_of[i] >= 0) { chosen[nch] = i; pos[nch++] = w.slot_of[i]; }
  if (nch < k) return MEC_ERR_READ_QUORUM;
  return MEC_OK;
}

// launch the rebuild of `targets` over blocks [first, first + nb) of raw shard files (arena position t at arena + t*fpitch, stride S
// between blocks, no frames) into out (block b, row q at (b*r + q)*pitch); the last of those blocks has shards of last_len bytes
static int launch_whole_rebuild(mec_codec* c, const uint8_t* arena, uint8_t* out, cudaStream_t st, const int* pos, int64_t fpitch,
                                int64_t S, int64_t last_len, int64_t first, int64_t nb, const uint8_t* rows, int r, int64_t pitch) {
  const int k = c->k;
  FusedDesc d;
  d.k = k; d.r = r; d.coef = rows; d.static_encode = false; d.contiguous = false; d.hash_outputs = false;
  d.key = kMagicKey; d.out_pitch = pitch; d.in_block_stride = S; d.digests = nullptr;
  const bool has_short = last_len != S;
  const int64_t nfull = has_short ? nb - 1 : nb;
  for (int pass = 0; pass < 2; pass++) {
    const int64_t f0 = pass == 0 ? 0 : nfull, cnt = pass == 0 ? nfull : nb - nfull;
    if (cnt <= 0) continue;
    d.nblocks = cnt;
    d.S = static_cast<int32_t>(pass == 0 ? S : last_len);
    for (int t = 0; t < k; t++) {
      const uint8_t* base = arena + pos[t] * fpitch;
      d.in_ptr[t] = base + (first + f0) * S;
      d.map_base[t] = base;
      d.map_len[t] = fpitch;
    }
    d.out = out + f0 * r * pitch;
    int rc = c->eng->launch_fused(d, c->opt, st);
    if (rc) return rc;
  }
  return MEC_OK;
}

extern "C" int64_t mec_decode_whole(mec_codec* c, const uint8_t* const* files, const uint8_t* sums, int64_t offset, int64_t length,
                                    int64_t total, uint8_t* dst, int* heal_hint) {
  NvtxRange nvtx("mec_decode_whole");
  if (heal_hint) *heal_hint = 0;
  if (!c || !files || !sums) return MEC_ERR_INVALID_ARGUMENT;
  if (offset < 0 || length < 0) return MEC_ERR_INVALID_ARGUMENT;      // cmd/erasure-decode.go:240-242
  if (offset + length > total) return MEC_ERR_INVALID_ARGUMENT;       // :243-245
  if (length == 0) return 0;                                          // :247-249
  if (!dst) return MEC_ERR_INVALID_ARGUMENT;
  std::lock_guard<std::mutex> lk(c->mu);
  int rc = require_whole(c);
  if (rc) return rc;
  const int k = c->k, n = c->n;
  if (k > kMaxK || n > kMaxShards || c->S() >= (1ll << 31)) return MEC_ERR_UNSUPPORTED;
  MEC_CUDA_OK(cudaSetDevice(c->device));
  const int64_t bs = c->block_size, S = c->S(), sfs = mec_shard_file_size(c, total);
  const ReadRange rr = read_range(c, offset, length, total);
  const int64_t nb = rr.nblocks;
  Slot& s = c->slots[0];
  SlotDrain drain(s);
  const int64_t fpitch = round_up(sfs, 16) + 256, pitch = round_up(S, 16);
  std::vector<uint8_t> alive(n), corrupt(n, 0);
  for (int i = 0; i < n; i++) alive[i] = files[i] != nullptr;
  int chosen[kMaxShards], pos[kMaxK];
  if ((rc = stage_verified_whole(c, files, sums, sfs, alive.data(), corrupt.data(), chosen, pos, fpitch, s))) return rc;
  DecodePlan p;
  if ((rc = plan_decode(c, chosen, k, nullptr, 1, &p))) return rc;
  const int r = p.r;
  if (r > 0) {
    if ((rc = s.out.ensure(static_cast<size_t>(nb * r * pitch)))) return rc;
    if ((rc = launch_whole_rebuild(c, static_cast<const uint8_t*>(s.aux.p), static_cast<uint8_t*>(s.out.p), s.st, pos, fpitch, S,
                                   rr.last_len, rr.start_block, nb, p.rows.data(), r, pitch)))
      return rc;
  }
  // writeDataBlocks by DMA: data shard i of block B sits in a verified shard file (stride S) or in a rebuilt row
  for (int i = 0; i < k; i++) {
    const uint8_t* base = nullptr;
    int64_t spitch = 0;
    for (int t = 0; t < k && !base; t++)
      if (chosen[t] == i) { base = static_cast<const uint8_t*>(s.aux.p) + pos[t] * fpitch + rr.start_block * S; spitch = S; }
    for (int q = 0; q < r && !base; q++)
      if (p.targets[q] == i) { base = static_cast<const uint8_t*>(s.out.p) + q * pitch; spitch = r * pitch; }
    if (!base) return MEC_ERR_UNEXPECTED;
    for (int64_t b = 0; b < nb; b++) {
      const DataSlice sl = data_slice(rr.start_block + b, i, b == nb - 1 ? rr.last_len : S, bs, total, offset, offset + length);
      if (sl.e > sl.a) {
        MEC_CUDA_OK(cudaMemcpyAsync(dst + (sl.a - offset), base + b * spitch + sl.off, static_cast<size_t>(sl.e - sl.a), cudaMemcpyDeviceToHost, s.st));
        c->st_d2h += sl.e - sl.a;
      }
    }
  }
  MEC_CUDA_OK(cudaStreamSynchronize(s.st));
  c->st_blocks_read += nb;
  c->st_shards_rebuilt += nb * r;
  if (heal_hint)
    for (int i = 0; i < n; i++)
      if (corrupt[i]) *heal_hint = MEC_ERR_FILE_CORRUPT;
  return length;
}

extern "C" int mec_heal_whole(mec_codec* c, const uint8_t* const* files, const uint8_t* sums, int64_t total,
                              uint8_t* const* out_files, uint8_t* out_sums, uint8_t* corrupt_out) {
  NvtxRange nvtx("mec_heal_whole");
  if (!c || !files || !sums || !out_files) return MEC_ERR_INVALID_ARGUMENT;
  if (corrupt_out) memset(corrupt_out, 0, static_cast<size_t>(c->n));
  if (total <= 0) return MEC_OK;
  std::lock_guard<std::mutex> lk(c->mu);
  int rc = require_whole(c);
  if (rc) return rc;
  const int k = c->k, n = c->n;
  if (k > kMaxK || n > kMaxShards || c->S() >= (1ll << 31)) return MEC_ERR_UNSUPPORTED;
  MEC_CUDA_OK(cudaSetDevice(c->device));
  const int64_t S = c->S(), sfs = mec_shard_file_size(c, total);
  const int64_t nblocks = ceil_frac(sfs, S), last_len = sfs - (nblocks - 1) * S;
  Slot& s = c->slots[0];
  SlotDrain drain(s);
  const int64_t fpitch = round_up(sfs, 16) + 256, pitch = round_up(S, 16);
  std::vector<uint8_t> alive(n), corrupt(n, 0), want(n);
  for (int i = 0; i < n; i++) { alive[i] = files[i] != nullptr; want[i] = out_files[i] != nullptr; }
  int chosen[kMaxShards], pos[kMaxK];
  if ((rc = stage_verified_whole(c, files, sums, sfs, alive.data(), corrupt.data(), chosen, pos, fpitch, s))) return rc;
  DecodePlan p;
  if ((rc = plan_decode(c, chosen, k, want.data(), 0, &p))) return rc;
  const int r = p.r;
  const int* targets = p.targets;
  if (r > 0) {
    if ((rc = s.out.ensure(static_cast<size_t>(nblocks * r * pitch)))) return rc;
    if ((rc = launch_whole_rebuild(c, static_cast<const uint8_t*>(s.aux.p), static_cast<uint8_t*>(s.out.p), s.st, pos, fpitch, S,
                                   last_len, 0, nblocks, p.rows.data(), r, pitch)))
      return rc;
    // rebuilt rows -> contiguous shard files on the device (for the whole-file hash), then files and sums go home
    if ((rc = s.src.ensure(static_cast<size_t>(r * fpitch + 256)))) return rc;
    if ((rc = s.dig.ensure(static_cast<size_t>((k + r) * 64)))) return rc;
    for (int q = 0; q < r; q++) {
      uint8_t* f = static_cast<uint8_t*>(s.src.p) + q * fpitch;
      const int64_t nfull = last_len == S ? nblocks : nblocks - 1;
      if (nfull > 0)
        MEC_CUDA_OK(cudaMemcpy2DAsync(f, static_cast<size_t>(S), static_cast<uint8_t*>(s.out.p) + q * pitch, static_cast<size_t>(r * pitch),
                                      static_cast<size_t>(S), static_cast<size_t>(nfull), cudaMemcpyDeviceToDevice, s.st));
      if (nfull < nblocks)
        MEC_CUDA_OK(cudaMemcpyAsync(f + nfull * S, static_cast<uint8_t*>(s.out.p) + (nfull * r + q) * pitch, static_cast<size_t>(last_len),
                                    cudaMemcpyDeviceToDevice, s.st));
      MEC_CUDA_OK(cudaMemsetAsync(f + sfs, 0, 256, s.st));
    }
    if ((rc = whole_hash_device(c, c->algo, static_cast<const uint8_t*>(s.src.p), fpitch, sfs, r, static_cast<uint8_t*>(s.dig.d.p) + k * 64, s.st))) return rc;
    c->eng->count_launch();
    for (int q = 0; q < r; q++) {
      MEC_CUDA_OK(cudaMemcpyAsync(out_files[targets[q]], static_cast<uint8_t*>(s.src.p) + q * fpitch, static_cast<size_t>(sfs), cudaMemcpyDeviceToHost, s.st));
      if (out_sums)
        MEC_CUDA_OK(cudaMemcpyAsync(out_sums + static_cast<size_t>(targets[q]) * 64, static_cast<uint8_t*>(s.dig.d.p) + (k + q) * 64, 64, cudaMemcpyDeviceToHost, s.st));
      c->st_d2h += sfs;
    }
  }
  // wanted shards that were read and verified are passed through
  for (int i = 0; i < n; i++)
    if (out_files[i] && p.present[i] && out_files[i] != files[i]) {
      memcpy(out_files[i], files[i], static_cast<size_t>(sfs));
      if (out_sums) memcpy(out_sums + static_cast<size_t>(i) * 64, sums + static_cast<size_t>(i) * 64, 64);
    }
  MEC_CUDA_OK(cudaStreamSynchronize(s.st));
  c->st_blocks_read += nblocks;
  c->st_shards_rebuilt += nblocks * r;
  bool any = false;
  for (int i = 0; i < n; i++) { any |= corrupt[i] != 0; if (corrupt_out) corrupt_out[i] = corrupt[i]; }
  return any ? MEC_ERR_FILE_CORRUPT : MEC_OK;  // Heal's derr (cmd/erasure-decode.go:338-341,366)
}

// Data movement between pools for a part written with a whole-file bitrot algorithm: Erasure.Decode over wholeBitrotReaders on
// `src` (as mec_decode_whole, with mec_decode_prefer's `prefer`) piped into Erasure.Encode on `dst` (as mec_transcode), without
// the object leaving the device.  wholeBitrotReader verifies a file before it hands out any byte of it (cmd/bitrot-whole.go:66-81),
// so the chosen readers' shard files are staged in slot 0's arena and hashed first — ONE whole_hash_kernel launch per round of
// readers — and nothing is written until k of them have verified.  The part then runs in chunks of source blocks through the
// codecs' slots, each on the source slot's stream: the missing data shards are rebuilt from the raw shard rows, whole_resplit_kernel
// re-splits the chunk into dst's object bytes, dst encodes them and its frames go out, so the copy back of chunk c overlaps the
// rebuild, re-split and encode of chunk c+1.
extern "C" int64_t mec_transcode_whole(mec_codec* src, const uint8_t* const* files, const uint8_t* sums, const uint8_t* prefer,
                                       int64_t total, mec_codec* dst, uint8_t* const* out_files, int write_quorum, int* heal_hint) {
  NvtxRange nvtx("mec_transcode_whole");
  if (heal_hint) *heal_hint = 0;
  if (!src || !dst || src == dst || !files || !sums || !out_files || total < 0) return MEC_ERR_INVALID_ARGUMENT;
  const bool whole_src = src->algo == MEC_SHA256 || src->algo == MEC_HIGHWAYHASH256 || src->algo == MEC_BLAKE2B512;
  if (!whole_src || dst->algo != MEC_HIGHWAYHASH256S || src->block_size % dst->block_size != 0 || src->device != dst->device)
    return MEC_ERR_UNSUPPORTED;
  int online = 0;
  for (int i = 0; i < dst->n; i++) online += out_files[i] != nullptr;
  if (online < write_quorum) return MEC_ERR_WRITE_QUORUM;  // cmd/erasure-encode.go:59-65
  if (total == 0) return 0;
  const int k = src->k, n = src->n;
  if (k > kMaxK || n > kMaxShards || src->S() >= (1ll << 31) || dst->S() >= (1ll << 31)) return MEC_ERR_UNSUPPORTED;
  int rc;
  if ((rc = require_streaming(dst))) return rc;
  std::scoped_lock lk(src->mu, dst->mu);  // two threads moving parts in opposite directions lock in the same order
  if ((rc = require_whole(src))) return rc;
  MEC_CUDA_OK(cudaSetDevice(src->device));
  const int64_t bs = src->block_size, S = src->S(), sfs = mec_shard_file_size(src, total);
  const int64_t nblocks = ceil_frac(total, bs), last_len = sfs - (nblocks - 1) * S;
  const int64_t fpitch = round_up(sfs, 16) + 256, pitch = round_up(S, 16);
  SlotDrain drain(src);
  Slot& s0 = src->slots[0];
  std::vector<uint8_t> alive(n), corrupt(n, 0);
  for (int i = 0; i < n; i++) alive[i] = files[i] != nullptr;
  int chosen[kMaxShards], pos[kMaxK];
  if ((rc = stage_verified_whole(src, files, sums, sfs, alive.data(), corrupt.data(), chosen, pos, fpitch, s0, prefer, true)))
    return rc;
  DecodePlan p;
  if ((rc = plan_decode(src, chosen, k, nullptr, 1, &p))) return rc;
  const int r = p.r;
  WholeResplitParams rp = {};
  rp.arena = static_cast<const uint8_t*>(s0.aux.p); rp.fpitch = fpitch; rp.pitch = pitch;
  rp.bs = bs; rp.S = S; rp.total = total; rp.k = k; rp.r = r;
  for (int t = 0; t < k; t++)
    if (chosen[t] < k) rp.src[chosen[t]] = static_cast<int8_t>(pos[t]);
  for (int q = 0; q < r; q++) rp.src[p.targets[q]] = static_cast<int8_t>(-1 - q);
  // ~32 MiB of object bytes per chunk; a shorter part is cut into about four chunks so that its copies back still overlap
  int64_t chunk = std::max<int64_t>(1, (32ll << 20) / bs);
  if (nblocks < 4 * chunk) chunk = ceil_frac(nblocks, 4);
  if (src->opt.chunk_blocks > 0) chunk = src->opt.chunk_blocks;
  const int64_t ebs = dst->block_size, epitch = round_up(dst->S(), 16);
  EncChunk inflight[kSlots];
  SlotRing ring(src, [&](int q) {
    frames_retire(dst, inflight[q], out_files, true, nullptr);
    dst->st_blocks_encoded += inflight[q].nb;
  });
  for (int64_t b0 = 0; b0 < nblocks; b0 += chunk) {
    if ((rc = ring.acquire())) return rc;
    const int si = ring.si;
    Slot& s = src->slots[si];
    Slot& d = dst->slots[si];
    const int64_t nb = std::min(chunk, nblocks - b0), bytes = std::min(total - b0 * bs, nb * bs), enb = ceil_frac(bytes, ebs);
    if (r > 0) {
      if ((rc = s.out.ensure(static_cast<size_t>(nb * r * pitch + 256)))) return rc;  // whole_resplit_kernel reads past the last row
      const int64_t chunk_last = b0 + nb == nblocks ? last_len : S;
      if ((rc = launch_whole_rebuild(src, rp.arena, static_cast<uint8_t*>(s.out.p), s.st, pos, fpitch, S, chunk_last, b0, nb,
                                     p.rows.data(), r, pitch)))
        return rc;
    }
    if ((rc = d.src.ensure(static_cast<size_t>(round_up(bytes, 16) + 256)))) return rc;
    if ((rc = d.out.ensure(static_cast<size_t>(enb * std::max(dst->m, 1) * epitch)))) return rc;
    if ((rc = d.dig.ensure(static_cast<size_t>(enb * dst->n * 32)))) return rc;
    rp.obj = static_cast<uint8_t*>(d.src.p);
    rp.rebuilt = static_cast<const uint8_t*>(s.out.p);
    rp.b0 = b0;
    whole_resplit_kernel<<<dim3(static_cast<unsigned>(nb), static_cast<unsigned>(k)), 128, 0, s.st>>>(rp);
    MEC_CUDA_OK(cudaGetLastError());
    src->eng->count_launch();
    if ((rc = encode_device_locked(dst, rp.obj, bytes, static_cast<uint8_t*>(d.out.p), epitch, static_cast<uint8_t*>(d.dig.d.p), s.st)))
      return rc;
    EncChunk& ec = inflight[si];
    ec = EncChunk{};
    ec.b0 = b0 * (bs / ebs); ec.nb = enb; ec.nfull = bytes / ebs; ec.tail = bytes % ebs; ec.s = &d; ec.pitch = epitch; ec.st = s.st;
    ec.d_src = rp.obj; ec.d_src_tail = rp.obj + ec.nfull * ebs;
    ec.d_out = static_cast<uint8_t*>(d.out.p); ec.d_out_tail = ec.d_out + ec.nfull * dst->m * epitch;
    ec.h_dig = static_cast<const uint8_t*>(d.dig.h.p); ec.h_dig_tail = ec.h_dig + ec.nfull * dst->n * 32;
    if ((rc = frames_enqueue_chunk(dst, ec, out_files, true, nullptr))) return rc;
    ring.submitted();
  }
  if ((rc = ring.finish())) return rc;
  src->st_blocks_read += nblocks;
  src->st_shards_rebuilt += nblocks * r;
  if (heal_hint)
    for (int i = 0; i < n; i++)
      if (corrupt[i]) *heal_hint = MEC_ERR_FILE_CORRUPT;
  return total;
}

// ------------------------------------------------------------------------------------------------
// Decode / Heal over a part whose drives mix bitrot formats.  healObject heals a legacy part into the streaming format
// (cmd/erasure-healing.go:593-596, a healed drive has no checksum entry and reads as HighwayHash256S, cmd/erasure-metadata.go:43-51),
// so after the first heal some drives hold [digest][shard] frames and the others raw shard files with whole-file sums, and every
// reader is opened with its own drive's algorithm (cmd/erasure-object.go:381-384, cmd/bitrot.go:112-117).  Both kinds run through
// reconstruct_range: streaming readers are staged and checked frame by frame, whole-file readers are hashed when first chosen.

// The read drives' formats.  Refuses an algos[i] that is no MEC_* value and a NULL sums beside a whole-file read drive
// (MEC_ERR_INVALID_ARGUMENT), and two whole-file algorithms (MEC_ERR_UNSUPPORTED: one legacy part has one).  *walgo = that
// algorithm, 0 when every read drive streams.  A drive is read where files[i] != NULL and, for heal, out_files[i] == NULL.
static int mixed_formats(const mec_codec* c, const int* algos, const uint8_t* const* files, uint8_t* const* out_files, const uint8_t* sums,
                         int* walgo) {
  int wa = 0;
  bool two = false;
  for (int i = 0; i < c->n; i++) {
    if (!files[i] || (out_files && out_files[i])) continue;
    const int a = algos[i];
    if (a < MEC_SHA256 || a > MEC_BLAKE2B512) return MEC_ERR_INVALID_ARGUMENT;
    if (a == MEC_HIGHWAYHASH256S) continue;
    if (wa && a != wa) two = true;
    if (!wa) wa = a;
  }
  if (wa && !sums) return MEC_ERR_INVALID_ARGUMENT;
  if (two) return MEC_ERR_UNSUPPORTED;
  *walgo = wa;
  return MEC_OK;
}

// reconstruct_range with the whole-file side when a read drive is whole-file (walgo != 0): its verified files sit in the codec's
// own buffer (c->whole) for the whole call.  alive[] must be set: only alive drives are ever read.
static int mixed_range(mec_codec* c, const int* algos, const uint8_t* const* files, const uint8_t* sums, int walgo, int64_t total,
                       const uint8_t* const* frames, const FrameGeom& g, const uint8_t* want, int data_only, const RangeSink& sk,
                       uint8_t* corrupt, uint8_t* alive, const uint8_t* prefer, bool hash_outputs) {
  if (!walgo) return reconstruct_range(c, frames, g, want, data_only, sk, corrupt, alive, prefer, hash_outputs);
  const int k = c->k, n = c->n;
  if (k > kMaxK || n > kMaxShards) return MEC_ERR_UNSUPPORTED;
  MEC_CUDA_OK(cudaSetDevice(c->device));
  const int64_t sfs = mec_shard_file_size(c, total), fpitch = round_up(sfs, 16) + 256;
  int rc;
  if ((rc = c->whole.ensure(static_cast<size_t>(k * fpitch + 256)))) return rc;
  if ((rc = c->whole_dig.ensure(static_cast<size_t>(k * 64)))) return rc;
  uint8_t whole[kMaxShards] = {};
  for (int i = 0; i < n; i++) whole[i] = alive[i] && algos[i] != MEC_HIGHWAYHASH256S;
  WholeSet w{files, sums, whole, walgo, sfs, fpitch, static_cast<uint8_t*>(c->whole.p), static_cast<uint8_t*>(c->whole_dig.d.p),
             static_cast<uint8_t*>(c->whole_dig.h.p), {}};
  for (int i = 0; i < n; i++) w.slot_of[i] = -1;
  return reconstruct_range(c, frames, g, want, data_only, sk, corrupt, alive, prefer, hash_outputs, &w);
}

extern "C" int64_t mec_decode_mixed(mec_codec* c, const int* algos, const uint8_t* const* files, const uint8_t* sums, const uint8_t* prefer,
                                    int64_t offset, int64_t length, int64_t total, uint8_t* dst, int* heal_hint) {
  NvtxRange nvtx("mec_decode_mixed");
  if (heal_hint) *heal_hint = 0;
  if (!c || !algos || !files) return MEC_ERR_INVALID_ARGUMENT;
  if (offset < 0 || length < 0) return MEC_ERR_INVALID_ARGUMENT;      // cmd/erasure-decode.go:240-242
  if (offset + length > total) return MEC_ERR_INVALID_ARGUMENT;       // :243-245
  if (length == 0) return 0;                                          // :247-249
  if (!dst) return MEC_ERR_INVALID_ARGUMENT;
  int walgo = 0;
  int rc = mixed_formats(c, algos, files, nullptr, sums, &walgo);
  if (rc) return rc;
  if ((rc = require_streaming(c))) return rc;
  std::lock_guard<std::mutex> lk(c->mu);
  const int k = c->k, n = c->n;
  const int64_t bs = c->block_size, S = c->S();
  const ReadRange rr = read_range(c, offset, length, total);
  const FrameGeom g{rr.nblocks, S, rr.last_len};
  if (static_cast<int64_t>(k) * g.last_len < std::min(offset + length, total) - rr.last_block * bs) return MEC_ERR_SHORT_DATA;
  const int64_t foff = rr.start_block * (32 + S);
  std::vector<const uint8_t*> in(n);
  std::vector<uint8_t> alive(n), want(n, 0), corrupt(n, 0);
  for (int i = 0; i < n; i++) {
    alive[i] = files[i] != nullptr;
    in[i] = files[i] && algos[i] == MEC_HIGHWAYHASH256S ? files[i] + foff : files[i];  // a whole-file reader's pointer is only tested for NULL
  }
  for (int i = 0; i < k; i++) want[i] = 1;
  RangeSink sk;
  sk.dst = dst; sk.first_block = rr.start_block; sk.lo = offset; sk.hi = offset + length; sk.bs = bs; sk.total = total;
  rc = mixed_range(c, algos, files, sums, walgo, total, in.data(), g, want.data(), 1, sk, corrupt.data(), alive.data(), prefer, false);
  if (rc) return rc;
  if (heal_hint)
    for (int i = 0; i < n; i++)
      if (corrupt[i]) *heal_hint = MEC_ERR_FILE_CORRUPT;
  return length;
}

extern "C" int mec_heal_mixed(mec_codec* c, const int* algos, const uint8_t* const* files, const uint8_t* sums, const uint8_t* prefer,
                              int64_t total, uint8_t* const* out_files, uint8_t* corrupt) {
  NvtxRange nvtx("mec_heal_mixed");
  if (!c || !algos || !files || !out_files) return MEC_ERR_INVALID_ARGUMENT;
  if (corrupt) memset(corrupt, 0, static_cast<size_t>(c->n));
  int walgo = 0;
  int rc = mixed_formats(c, algos, files, out_files, sums, &walgo);
  if (rc) return rc;
  if (total <= 0) return MEC_OK;
  if ((rc = require_streaming(c))) return rc;
  std::lock_guard<std::mutex> lk(c->mu);
  const int n = c->n;
  const int64_t S = c->S(), sfs = mec_shard_file_size(c, total);
  FrameGeom g;
  g.nblocks = ceil_frac(total, c->block_size);
  g.S = S;
  g.last_len = sfs - (g.nblocks - 1) * S;
  std::vector<uint8_t> alive(n), want(n, 0), bad(n, 0);
  // healObject opens no reader on a drive it heals (cmd/erasure-healing.go:572-575): a stale drive is never read
  for (int i = 0; i < n; i++) { alive[i] = files[i] != nullptr && out_files[i] == nullptr; want[i] = out_files[i] != nullptr; }
  RangeSink sk;
  sk.out = out_files;
  rc = mixed_range(c, algos, files, sums, walgo, total, files, g, want.data(), 0, sk, bad.data(), alive.data(), prefer, true);
  if (rc) return rc;
  bool any = false;
  for (int i = 0; i < n; i++) { any |= bad[i] != 0; if (corrupt) corrupt[i] = bad[i]; }
  return any ? MEC_ERR_FILE_CORRUPT : MEC_OK;
}

// ------------------------------------------------------------------------------------------------
// shard-shaped low level calls
static int apply_rows_host(mec_codec* c, const uint8_t* rows, int r, const uint8_t* const* in, uint8_t* const* outp,
                           int64_t len, bool is_encode) {
  MEC_CUDA_OK(cudaSetDevice(c->device));
  Slot& s = c->slots[0];
  const int k = c->k;
  const int64_t ipitch = round_up(len, 256), opitch = round_up(len, 16);
  int rc;
  if ((rc = s.src.ensure(static_cast<size_t>(k * ipitch + 512)))) return rc;
  if ((rc = s.out.ensure(static_cast<size_t>(std::max(r, 1) * opitch)))) return rc;
  for (int t = 0; t < k; t++)
    MEC_CUDA_OK(cudaMemcpyAsync(static_cast<uint8_t*>(s.src.p) + t * ipitch, in[t], static_cast<size_t>(len),
                                cudaMemcpyHostToDevice, s.st));
  FusedDesc d;
  d.k = k; d.r = r; d.coef = rows; d.static_encode = is_encode; d.contiguous = false;
  d.nblocks = 1; d.S = static_cast<int32_t>(len); d.in_block_stride = 0;
  for (int t = 0; t < k; t++) {
    d.in_ptr[t] = static_cast<const uint8_t*>(s.src.p) + t * ipitch;
    d.map_base[t] = d.in_ptr[t];
    d.map_len[t] = ipitch;
  }
  d.out = static_cast<uint8_t*>(s.out.p); d.out_pitch = opitch; d.digests = nullptr; d.key = kMagicKey;
  if ((rc = c->eng->launch_fused(d, c->opt, s.st))) return rc;
  for (int q = 0; q < r; q++)
    MEC_CUDA_OK(cudaMemcpyAsync(outp[q], static_cast<uint8_t*>(s.out.p) + q * opitch, static_cast<size_t>(len),
                                cudaMemcpyDeviceToHost, s.st));
  MEC_CUDA_OK(cudaStreamSynchronize(s.st));
  return MEC_OK;
}

extern "C" int mec_rs_encode_shards(mec_codec* c, uint8_t* const* shards, int64_t len) {
  if (!c || !shards) return MEC_ERR_INVALID_ARGUMENT;
  if (len == 0) return MEC_ERR_SHARD_NO_DATA;
  if (len >= (1ll << 31) || c->k > kMaxK || c->m > kMaxR) return MEC_ERR_UNSUPPORTED;
  if (c->m == 0) return MEC_OK;
  std::lock_guard<std::mutex> lk(c->mu);
  if (int rc = ensure_engine(c)) return rc;
  return apply_rows_host(c, c->matrix.data() + static_cast<size_t>(c->k) * c->k, c->m, shards, shards + c->k, len, true);
}

extern "C" int mec_rs_reconstruct_shards(mec_codec* c, uint8_t* const* shards, const uint8_t* present, int64_t len,
                                         int data_only) {
  if (!c || !shards || !present) return MEC_ERR_INVALID_ARGUMENT;
  const int k = c->k, n = c->n;
  int np = 0;
  for (int i = 0; i < n; i++) np += present[i] != 0;
  if (np == 0 || len == 0) return MEC_ERR_SHARD_NO_DATA;
  if (np == n) return MEC_OK;
  if (np < k) return MEC_ERR_TOO_FEW_SHARDS;
  if (len >= (1ll << 31) || k > kMaxK) return MEC_ERR_UNSUPPORTED;
  // Reconstruct reads the first k present shards and rebuilds every missing one
  int chosen[kMaxShards], nch = 0;
  uint8_t want[kMaxShards];
  for (int i = 0; i < n; i++) {
    want[i] = !present[i];
    if (present[i] && nch < k) chosen[nch++] = i;
  }
  DecodePlan p;
  if (int rc = plan_decode(c, chosen, nch, want, data_only, &p)) return rc;
  const int r = p.r;
  if (r == 0) return MEC_OK;
  std::vector<const uint8_t*> in(k);
  std::vector<uint8_t*> outp(r);
  for (int t = 0; t < k; t++) in[t] = shards[chosen[t]];
  for (int q = 0; q < r; q++) outp[q] = shards[p.targets[q]];
  std::lock_guard<std::mutex> lk(c->mu);
  if (int rc = ensure_engine(c)) return rc;
  return apply_rows_host(c, p.rows.data(), r, in.data(), outp.data(), len, false);
}

extern "C" int mec_hh256_batch(mec_codec* c, const uint8_t* msgs, int64_t msg_len, int64_t count, uint8_t* digests) {
  if (!c || msg_len < 0 || count < 0) return MEC_ERR_INVALID_ARGUMENT;
  if (count == 0) return MEC_OK;
  if (msg_len >= (1ll << 31)) return MEC_ERR_UNSUPPORTED;
  std::lock_guard<std::mutex> lk(c->mu);
  int rc;
  if ((rc = ensure_engine(c))) return rc;
  MEC_CUDA_OK(cudaSetDevice(c->device));
  Slot& s = c->slots[0];
  if ((rc = s.dig.d.ensure(static_cast<size_t>(count * 32)))) return rc;
  const int64_t mp = std::max<int64_t>(round_up(msg_len, 16), 16);
  if ((rc = s.src.ensure(static_cast<size_t>(count * mp + 512)))) return rc;
  if (msg_len > 0)
    MEC_CUDA_OK(cudaMemcpy2DAsync(s.src.p, static_cast<size_t>(mp), msgs, static_cast<size_t>(msg_len),
                                  static_cast<size_t>(msg_len), static_cast<size_t>(count), cudaMemcpyHostToDevice, s.st));
  FusedDesc d;
  d.k = 1; d.r = 0; d.contiguous = false; d.key = kMagicKey;
  d.nblocks = count; d.S = static_cast<int32_t>(msg_len);
  d.in_block_stride = mp;
  d.in_ptr[0] = static_cast<const uint8_t*>(s.src.p);
  d.map_base[0] = d.in_ptr[0];
  d.map_len[0] = count * mp + 256;
  d.digests = static_cast<uint8_t*>(s.dig.d.p);
  if ((rc = c->eng->launch_fused(d, c->opt, s.st))) return rc;
  MEC_CUDA_OK(cudaMemcpyAsync(digests, s.dig.d.p, static_cast<size_t>(count * 32), cudaMemcpyDeviceToHost, s.st));
  MEC_CUDA_OK(cudaStreamSynchronize(s.st));
  return MEC_OK;
}

// ------------------------------------------------------------------------------------------------
// self tests (cmd/erasure-coding.go:149-205, cmd/bitrot.go:224-254)
static uint64_t xxh64(const uint8_t* p, size_t n) {
  const uint64_t P1 = 11400714785074694791ull, P2 = 14029467366897019727ull, P3 = 1609587929392839161ull,
                 P4 = 9650029242287828579ull, P5 = 2870177450012600261ull;
  auto rol = [](uint64_t x, int r) { return (x << r) | (x >> (64 - r)); };
  auto rd64 = [](const uint8_t* q) { uint64_t v; memcpy(&v, q, 8); return v; };
  auto rd32 = [](const uint8_t* q) { uint32_t v; memcpy(&v, q, 4); return static_cast<uint64_t>(v); };
  auto round = [&](uint64_t acc, uint64_t in) { acc += in * P2; acc = rol(acc, 31); return acc * P1; };
  auto merge = [&](uint64_t acc, uint64_t v) { acc ^= round(0, v); return acc * P1 + P4; };
  const uint8_t* end = p + n;
  uint64_t h;
  if (n >= 32) {
    uint64_t v1 = P1 + P2, v2 = P2, v3 = 0, v4 = 0 - P1;
    do {
      v1 = round(v1, rd64(p)); v2 = round(v2, rd64(p + 8)); v3 = round(v3, rd64(p + 16)); v4 = round(v4, rd64(p + 24));
      p += 32;
    } while (p + 32 <= end);
    h = rol(v1, 1) + rol(v2, 7) + rol(v3, 12) + rol(v4, 18);
    h = merge(h, v1); h = merge(h, v2); h = merge(h, v3); h = merge(h, v4);
  } else {
    h = P5;
  }
  h += n;
  while (p + 8 <= end) { h ^= round(0, rd64(p)); h = rol(h, 27) * P1 + P4; p += 8; }
  if (p + 4 <= end) { h ^= rd32(p) * P1; h = rol(h, 23) * P2 + P3; p += 4; }
  while (p < end) { h ^= (*p) * P5; h = rol(h, 11) * P1; p++; }
  h ^= h >> 33; h *= P2; h ^= h >> 29; h *= P3; h ^= h >> 32;
  return h;
}

extern "C" int mec_selftest(int device) {
  static const struct { uint8_t k, m; uint64_t want; } kGold[] = {  // cmd/erasure-coding.go:160
      {2, 2, 0x23fb21be2496f5d3ull}, {2, 3, 0xa5cd5600ba0d8e7cull}, {3, 1, 0x60ab052148b010b4ull}, {3, 2, 0xe64927daef76435aull},
      {3, 3, 0x672f6f242b227b21ull}, {3, 4, 0x571e41ba23a6dc6ull}, {4, 1, 0x524eaa814d5d86e2ull}, {4, 2, 0x62b9552945504fefull},
      {4, 3, 0xcbf9065ee053e518ull}, {4, 4, 0x9a07581dcd03da8ull}, {4, 5, 0xbf2d27b55370113full}, {5, 1, 0xf71031a01d70dafull},
      {5, 2, 0x8e5845859939d0f4ull}, {5, 3, 0x7ad9161acbb4c325ull}, {5, 4, 0xc446b88830b4f800ull}, {5, 5, 0xabf1573cc6f76165ull},
      {5, 6, 0x7b5598a85045bfb8ull}, {6, 1, 0xe2fc1e677cc7d872ull}, {6, 2, 0x7ed133de5ca6a58eull}, {6, 3, 0x39ef92d0a74cc3c0ull},
      {6, 4, 0xcfc90052bc25d20ull}, {6, 5, 0x71c96f6baeef9c58ull}, {6, 6, 0x4b79056484883e4cull}, {6, 7, 0xb1a0e2427ac2dc1aull},
      {7, 1, 0x937ba2b7af467a22ull}, {7, 2, 0x5fd13a734d27d37aull}, {7, 3, 0x3be2722d9b66912full}, {7, 4, 0x14c628e59011be3dull},
      {7, 5, 0xcc3b39ad4c083b9full}, {7, 6, 0x45af361b7de7a4ffull}, {7, 7, 0x456cc320cec8a6e6ull}, {7, 8, 0x1867a9f4db315b5cull},
      {8, 1, 0xbc5756b9a9ade030ull}, {8, 2, 0xdfd7d9d0b3e36503ull}, {8, 3, 0x72bb72c2cdbcf99dull}, {8, 4, 0x3ba5e9b41bf07f0ull},
      {8, 5, 0xd7dabc15800f9d41ull}, {8, 6, 0xb482a6169fd270full}, {8, 7, 0x50748e0099d657e8ull}, {9, 1, 0xc77ae0144fcaeb6eull},
      {9, 2, 0x8a86c7dbebf27b68ull}, {9, 3, 0xa64e3be6d6fe7e92ull}, {9, 4, 0x239b71c41745d207ull}, {9, 5, 0x2d0803094c5a86ceull},
      {9, 6, 0xa3c2539b3af84874ull}, {10, 1, 0x7d30d91b89fcec21ull}, {10, 2, 0xfa5af9aa9f1857a3ull}, {10, 3, 0x84bc4bda8af81f90ull},
      {10, 4, 0x6c1cba8631de994aull}, {10, 5, 0x4383e58a086cc1acull}, {11, 1, 0x4ed2929a2df690bull}, {11, 2, 0xecd6f1b1399775c0ull},
      {11, 3, 0xc78cfbfc0dc64d01ull}, {11, 4, 0xb2643390973702d6ull}, {12, 1, 0x3b2a88686122d082ull}, {12, 2, 0xfd2f30a48a8e2e9ull},
      {12, 3, 0xd5ce58368ae90b13ull}, {13, 1, 0x9c88e2a9d1b8fff8ull}, {13, 2, 0xcb8460aa4cf6613ull}, {14, 1, 0x78a28bbaec57996eull}};
  uint8_t test[256];
  for (int i = 0; i < 256; i++) test[i] = static_cast<uint8_t>(i);
  for (const auto& g : kGold) {
    mec_codec* c = nullptr;
    int rc = mec_codec_new(g.k, g.m, 1 << 20, MEC_HIGHWAYHASH256S, device, &c);
    if (rc) return rc;
    const int n = g.k + g.m;
    const int64_t per = ceil_frac(256, g.k);
    std::vector<uint8_t> store(static_cast<size_t>(n * per), 0);
    memcpy(store.data(), test, 256);  // Split: zero padded
    std::vector<uint8_t*> sh(n);
    for (int i = 0; i < n; i++) sh[i] = store.data() + i * per;
    rc = mec_rs_encode_shards(c, sh.data(), per);
    if (rc) { mec_codec_free(c); return rc; }
    std::vector<uint8_t> buf;
    for (int i = 0; i < n; i++) { buf.push_back(static_cast<uint8_t>(i)); buf.insert(buf.end(), sh[i], sh[i] + per); }
    if (xxh64(buf.data(), buf.size()) != g.want) {
      set_last_error("erasure self-test mismatch for d:" + std::to_string(g.k) + " p:" + std::to_string(g.m));
      mec_codec_free(c);
      return MEC_ERR_UNEXPECTED;
    }
    std::vector<uint8_t> first(sh[0], sh[0] + per), present(n, 1);
    memset(sh[0], 0xee, static_cast<size_t>(per));
    present[0] = 0;
    rc = mec_rs_reconstruct_shards(c, sh.data(), present.data(), per, 1);
    if (rc == 0 && memcmp(first.data(), sh[0], static_cast<size_t>(per)) != 0) rc = MEC_ERR_UNEXPECTED;
    mec_codec_free(c);
    if (rc) { set_last_error("erasure self-test: first-shard reconstruct failed"); return rc; }
  }
  // bitrot self-test: HighwayHash chain (cmd/bitrot.go:228): msg grows by its own digest
  {
    mec_codec* c = nullptr;
    int rc = mec_codec_new(2, 2, 1 << 20, MEC_HIGHWAYHASH256S, device, &c);
    if (rc) return rc;
    static const uint8_t want[32] = {0x39, 0xc0, 0x40, 0x7e, 0xd3, 0xf0, 0x1b, 0x18, 0xd2, 0x2c, 0x85, 0xdb, 0x4a, 0xef, 0xf1, 0x1e,
                                     0x06, 0x0c, 0xa5, 0xf4, 0x31, 0x31, 0xb0, 0x12, 0x67, 0x31, 0xca, 0x19, 0x7c, 0xd4, 0x23, 0x13};
    std::vector<uint8_t> msg;
    uint8_t sum[32];
    for (int i = 0; i < 32 * 32; i += 32) {
      rc = mec_hh256_batch(c, msg.data(), static_cast<int64_t>(msg.size()), 1, sum);
      if (rc) { mec_codec_free(c); return rc; }
      msg.insert(msg.end(), sum, sum + 32);
    }
    mec_codec_free(c);
    if (memcmp(sum, want, 32) != 0) { set_last_error("bitrot self-test mismatch"); return MEC_ERR_UNEXPECTED; }
  }
  // the whole-file algorithms of the same self test (cmd/bitrot.go:225-229): Size()*BlockSize() bytes, Size() at a time
  {
    static const struct { int algo, size, block; const char* want; } kChains[] = {
        {MEC_SHA256, 32, 64, "a7677ff19e0182e4d52e3a3db727804abc82a5818749336369552e54b838b004"},
        {MEC_BLAKE2B512, 64, 128, "e519b7d84b1c3c917985f544773a35cf265dcab10948be3550320d156bab612124a5ae2ae5a8c73c0eea360f68b0e28136f26e858756dbfe7375a7389f26c669"},
        {MEC_HIGHWAYHASH256, 32, 32, "39c0407ed3f01b18d22c85db4aeff11e060ca5f43131b0126731ca197cd42313"}};
    for (const auto& ch : kChains) {
      mec_codec* c = nullptr;
      int rc = mec_codec_new(2, 2, 1 << 20, ch.algo, device, &c);
      if (rc) return rc;
      std::vector<uint8_t> msg;
      uint8_t sum[64];
      for (int i = 0; i < ch.size * ch.block; i += ch.size) {
        rc = mec_whole_hash(c, ch.algo, msg.data(), static_cast<int64_t>(msg.size()), 1, sum);
        if (rc) { mec_codec_free(c); return rc; }
        msg.insert(msg.end(), sum, sum + ch.size);
      }
      mec_codec_free(c);
      for (int i = 0; i < ch.size; i++) {
        unsigned v = 0;
        sscanf(ch.want + 2 * i, "%2x", &v);
        if (sum[i] != v) { set_last_error("bitrot self-test mismatch (whole-file algorithm " + std::to_string(ch.algo) + ")"); return MEC_ERR_UNEXPECTED; }
      }
    }
  }
  return MEC_OK;
}

// ------------------------------------------------------------------------------------------------
// Cross-request coalescer.  MinIO builds one Erasure per request (cmd/erasure-object.go:1371) and encodes ONE block per loop
// iteration (cmd/erasure-encode.go:76-108) on thousands of concurrent request goroutines (cmd/handler-api.go:139-143).  A GPU
// launch that carries one 1 MiB block keeps one CTA busy on one of 132 SMs (H100) for as long as a launch of a thousand blocks takes.
// The batcher turns concurrency into batch size: callers block in mec_batcher_encode*, a worker thread merges whatever is
// queued (same k, m, block size by construction) into ONE staged buffer, ONE launch over all full blocks (plus one small
// launch per short tail block), and one pass of DMA back into every caller's own frames; up to six merged batches are in
// flight on the codec's six slots, so staging, kernel and copy-back of consecutive batches overlap.
#include <chrono>
#include <condition_variable>
#include <deque>
#include <unordered_map>

// PutObject (encode), GetObject (decode), Heal, a move between pools, a move of a part written with a whole-file bitrot algorithm,
// bitrot verification of a drive's parts (VerifyFile)
enum class ReqKind { Put, Get, Heal, Transcode, TranscodeWhole, Verify };
// a GET, heal or move: stages its readers, and digest verdicts (per frame; per shard file for a whole-file move) decide which of
// its requests are done
static inline bool is_read(ReqKind k) { return k != ReqKind::Put && k != ReqKind::Verify; }
static inline bool is_move(ReqKind k) { return k == ReqKind::Transcode || k == ReqKind::TranscodeWhole; }

struct BatchReq {
  ReqKind kind = ReqKind::Put;
  // GET, heal and transcode (a heal and a transcode read the whole part: offset 0, length = total)
  const uint8_t* const* gfiles = nullptr;
  int64_t offset = 0, length = 0, total = 0;
  uint8_t* dst = nullptr;
  int* heal_hint = nullptr;
  uint64_t alive_mask = 0;           // bit i = reader i is online (heal, GET with `prefer`: one of the k chosen readers)
  int64_t get_slot0 = 0, get_tail_slot = -1, get_nblocks = 0;  // placement of the request's blocks in the merged batch
  const uint8_t* prefer = nullptr;   // preferReaders (cmd/erasure-decode.go:92-123), for the redo of a request that met bitrot
  // whole-file move, or a mixed GET / heal with a whole-file reader among its k chosen: the part's algorithm (0 for every other
  // request: a batch holds one algorithm), the expected digests (+ i*64) and the chosen whole-file readers (bit i = drive i)
  int whole_algo = 0;
  const uint8_t* whole_sums = nullptr;
  uint64_t whole_drives = 0;
  // mec_batcher_decode_mixed / _heal_mixed: every drive's bitrot algorithm; the private path is mec_decode_mixed / mec_heal_mixed
  const int* algos = nullptr;
  // heal
  uint8_t* const* outs = nullptr;
  uint8_t* corrupt = nullptr;
  uint64_t stale_mask = 0;           // bit i = out_files[i] != NULL: heals share a launch only with the same stale drives
  // PUT, and the destination side of a transcode (len = total, files = out_files, with_data): both laid out by put_layout
  const uint8_t* src = nullptr;
  int64_t len = 0;
  uint8_t* const* files = nullptr;
  uint8_t* data_digests = nullptr;
  bool with_data = false;
  bool mapped = false;   // every buffer of the call is page-locked (device-addressable): eligible for the gather / scatter kernels
  int crc_which = 0;          // MEC_CRC* mask of mec_batcher_encode_crc / _sums; the results go to crc_out[0..3)
  uint64_t* crc_out = nullptr;
  int sum_which = 0;          // MEC_SUM_* mask of mec_batcher_encode_sums; the digests go to their slots of sums[0..MEC_SUM_BYTES)
  uint8_t* sums = nullptr;
  // verify (mec_batcher_verify): the call's parts, decided on the caller's thread (verify_decide: results[p] == MEC_OK with bytes to
  // hash marks a part the batch hashes); its streaming frames, whole-file parts and staged bytes (verify_staged)
  int64_t vparts = 0, vframes = 0, vwhole = 0, vbytes = 0;
  const int* valgos = nullptr;
  const uint8_t* const* vfiles = nullptr;
  const int64_t* vfile_lens = nullptr;
  const int64_t* vpart_lens = nullptr;
  const uint8_t* vsums = nullptr;
  int* vresults = nullptr;
  // mec_batcher_encode_sse / _decode_sse: the stream's key (and a PUT's nonce), read by the worker while the caller waits; the
  // plaintext bytes of a PUT (len is its ciphertext), the plaintext range and size of a GET (offset / length / total are the
  // ciphertext range of its whole packages); where the batch placed its ciphertext and its first package row
  const uint8_t* sse_key = nullptr;
  const uint8_t* sse_nonce = nullptr;
  int64_t sse_offset = 0, sse_len = 0, sse_total = 0;
  int64_t sse_ct = 0, sse_row0 = 0;
  int sse_chacha = 0;  // the batcher's option "dare_chacha20" when the request was admitted (mec_batcher_set_option)
  int64_t result = 0;
  bool done = false;
  std::condition_variable cv;  // one per request: a finished batch wakes its own callers, not every thread parked in the batcher
  EncChunk ch;   // placement inside the merged batch
};

// The decode plan of one erasure pattern of merged reads: the host plan and the latency kernel's per-block table entry
struct BatchPattern {
  DecodePlan plan;
  SmallPattern sp;
};
constexpr size_t kMaxCachedPatterns = 4096;

// The environment switches of the coalescer's staging and output paths, read once per batcher by batcher_create
struct BatcherSwitches {
  bool memcpy = false;     // MEC_BATCHER_MEMCPY: PUTs take the copy-engine path, reads and moves the private handles
  bool gather = false;     // MEC_BATCHER_GATHER: the gather kernel stages every PUT
  int gather_pct = 0;      // MEC_BATCHER_GATHER_PCT (0-100): that share of a PUT batch is staged by the gather kernel on `aux`
  int64_t dma_blocks = 1;  // MEC_BATCHER_DMA_BLOCKS: reads of fewer blocks are staged by the gather kernel
  int get_out = 0;         // MEC_BATCHER_GET_OUT: how merged GETs reach the callers' buffers (batcher_submit_get)
  int depth = 4;           // MEC_BATCHER_DEPTH: batches the worker aims to keep in flight (0: cut batches at max_batch_blocks only)
  bool trace = false;      // MEC_BATCHER_TRACE: device phase times of every kernel batch (mec_batcher_stat "us_stage", ...)
};

struct mec_batcher {
  mec_codec* codec = nullptr;
  mec_codec* serial = nullptr;       // private handle for calls that cannot ride in a batch (pageable buffers, bitrot fail-over)
  std::mutex serial_mu;
  int64_t max_blocks = 256;
  int max_wait_us = 200;
  std::mutex mu;
  std::condition_variable cv_work, cv_done;
  std::deque<BatchReq*> queue;
  bool stop = false;
  std::thread worker;
  std::atomic<int64_t> st_batches{0}, st_requests{0}, st_blocks{0}, st_kernel_batches{0};
  std::atomic<int64_t> st_redone{0};  // merged GETs and heals that met a frame failing its digest and were redone on their own
  std::atomic<int64_t> st_crc_requests{0};  // PUTs that got their object checksums (mec_batcher_encode_crc)
  std::atomic<int64_t> st_sum_requests{0};  // PUTs that got at least one object hash (mec_batcher_encode_sums)
  // object hashes of a PUT batch run on a second stream per slot, forked once the batch is staged (ev_staged) and joined before the
  // slot's stream ends (ev_summed), so the batch's encode is not queued behind them
  Stream sum_st[kSlots];
  Event ev_staged[kSlots], ev_summed[kSlots];
  // MEC_BATCHER_MIX_PATTERNS (and a codec whose options allow the latency kernel): GETs merge with GETs and heals with heals
  // whatever their reader and stale sets, as long as a batch of several erasure patterns fits one latency launch
  bool mix = false;
  std::atomic<int64_t> st_patterns{0}, st_mixed{0};  // distinct patterns summed over read batches; read batches of more than one
  // decode plans by (reader mask, target mask), owned by the worker thread: a steady workload inverts no matrix
  std::unordered_map<uint64_t, BatchPattern> patterns;
  BatcherSwitches sw;
  // hybrid staging (sw.gather_pct): part of a batch is read by the gather kernel on `aux` while the copy engine moves the rest
  Stream aux;
  Event ev_table[kSlots], ev_gather[kSlots];
  // where the worker's time and each batch's stream time go (mec_batcher_stat "us_*"); device phases need sw.trace
  Event ev_ph[kSlots][4];
  std::atomic<int64_t> us_submit{0}, us_sync{0}, us_finish{0}, us_idle{0}, us_stage{0}, us_kernel{0}, us_scatter{0};
  // mec_batcher_new_transcode: the destination codec of merged moves (private; its slot i carries the destination side of the batch
  // on source slot i), and the destination half of the private pair for moves that cannot ride in a batch (with `serial`)
  mec_codec* dst = nullptr;
  mec_codec* serial_dst = nullptr;
  std::atomic<int64_t> st_transcodes{0}, st_transcodes_serial{0};  // moves completed by merged batches / by the private pair
  // mec_batcher_transcode_whole: the source halves of the private pair, one per whole-file algorithm (SHA256, HighwayHash256,
  // BLAKE2b512), each created on first use, and the moves completed by merged batches / by the private pair
  mec_codec* serial_whole[3] = {};
  std::atomic<int64_t> st_transcodes_whole{0}, st_transcodes_whole_serial{0};
  // mec_batcher_decode_mixed / _heal_mixed: calls with a whole-file reader completed by merged batches, and mixed calls of the
  // private path (redos included)
  std::atomic<int64_t> st_reads_whole{0}, st_reads_whole_serial{0};
  // mec_batcher_verify: calls completed by merged batches / by the private handle
  std::atomic<int64_t> st_verifies{0}, st_verifies_serial{0};
  // mec_batcher_encode_sse / _decode_sse: calls completed by merged batches, and calls of the private path (redos included)
  std::atomic<int64_t> st_sse_puts{0}, st_sse_gets{0}, st_sse_serial{0};
  std::atomic<int> dare_chacha20{0};  // mec_batcher_set_option: recorded by every encrypted request as it is admitted
  // the batcher owns its codecs; each drains its slots before it is freed.  The worker has been joined (mec_batcher_free) or
  // never started (batcher_create's failures).
  ~mec_batcher() {
    for (mec_codec* h : {serial, serial_dst, serial_whole[0], serial_whole[1], serial_whole[2], dst, codec}) mec_codec_free(h);
  }
};

namespace {
struct InflightBatch {
  std::vector<BatchReq*> reqs;
  ReqKind kind = ReqKind::Put;
  bool needs_retire = true;  // false: the scatter kernel already assembled the frames
  bool traced = false;
};

// The private handle `h` of `g`'s geometry and bitrot algorithm `algo`, created on first use
static mec_codec* batcher_private(mec_batcher* b, const mec_codec* g, mec_codec*& h, int algo = MEC_HIGHWAYHASH256S) {
  std::lock_guard<std::mutex> lk(b->serial_mu);
  if (!h) {
    mec_codec* p = nullptr;
    if (mec_codec_new(g->k, g->m, g->block_size, algo, g->device, &p) == MEC_OK) h = p;
    if (p && &h == &b->serial) p->dare_chacha20 = b->dare_chacha20.load();
  }
  return h;
}
// index of a whole-file algorithm in mec_batcher::serial_whole
static inline int whole_index(int algo) { return algo == MEC_SHA256 ? 0 : algo == MEC_HIGHWAYHASH256 ? 1 : 2; }

// A read or move on its own, through the private handles: a call the merged path cannot take, or the redo of a merged one that met
// a frame failing its digest, which applies parallelReader's block-sequential fail-over exactly (a heal rewrites every out file in
// full and reports the failing readers; a transcode rewrites every out file in full through mec_transcode on the private pair, its
// write quorum already checked on the caller's thread; a whole-file move does the same through mec_transcode_whole, whose source
// handle carries the part's algorithm)
static int64_t batcher_run_alone(mec_batcher* b, const BatchReq& r) {
  if (r.sse_key) {  // an encrypted PUT or GET: mec_encode_sse / mec_decode_sse under the option it was admitted with, the write
                    // quorum already checked
    b->st_sse_serial++;
    mec_codec* sc = batcher_private(b, b->codec, b->serial);
    if (!sc) return MEC_ERR_UNEXPECTED;
    if (r.kind == ReqKind::Put) return encode_sse(sc, r.src, r.sse_len, r.sse_key, r.sse_nonce, r.files, 0, r.sse_chacha);
    return decode_sse(sc, r.gfiles, r.prefer, r.sse_offset, r.sse_len, r.total, r.sse_key, r.dst, r.heal_hint, r.sse_chacha);
  }
  if (r.kind == ReqKind::TranscodeWhole) {
    b->st_transcodes_whole_serial++;
    mec_codec* sc = batcher_private(b, b->codec, b->serial_whole[whole_index(r.whole_algo)], r.whole_algo);
    mec_codec* sd = batcher_private(b, b->dst, b->serial_dst);
    return sc && sd ? mec_transcode_whole(sc, r.gfiles, r.whole_sums, r.prefer, r.total, sd, r.files, 0, r.heal_hint) : MEC_ERR_UNEXPECTED;
  }
  if (r.kind == ReqKind::Transcode) b->st_transcodes_serial++;
  mec_codec* sc = batcher_private(b, b->codec, b->serial);
  if (r.algos) {  // a mixed read: fail-over may reach a drive of either format
    b->st_reads_whole_serial++;
    if (!sc) return MEC_ERR_UNEXPECTED;
    if (r.kind == ReqKind::Heal) return mec_heal_mixed(sc, r.algos, r.gfiles, r.whole_sums, r.prefer, r.total, r.outs, r.corrupt);
    return mec_decode_mixed(sc, r.algos, r.gfiles, r.whole_sums, r.prefer, r.offset, r.length, r.total, r.dst, r.heal_hint);
  }
  if (r.kind == ReqKind::Transcode) {
    mec_codec* sd = batcher_private(b, b->dst, b->serial_dst);
    return sc && sd ? mec_transcode(sc, r.gfiles, r.prefer, r.total, sd, r.files, 0, r.heal_hint) : MEC_ERR_UNEXPECTED;
  }
  if (!sc) return MEC_ERR_UNEXPECTED;
  if (r.kind == ReqKind::Heal) return mec_heal_prefer(sc, r.gfiles, r.prefer, r.total, r.outs, r.corrupt);
  return mec_decode_prefer(sc, r.gfiles, r.prefer, r.offset, r.length, r.total, r.dst, r.heal_hint);
}

// The stream-table position of the first whole-file part of each algorithm group (whole_group) in a merged verify batch: the table
// holds the SHA256 parts of every request, then the HighwayHash256 parts, then the BLAKE2b512 parts, each group in request order
// and part order within a request
static void verify_whole_firsts(const std::vector<BatchReq*>& reqs, int64_t (&first)[kWholeGroups]) {
  int64_t counts[kWholeGroups] = {};
  for (const BatchReq* r : reqs)
    for (int64_t p = 0; p < r->vparts; p++)
      if (r->vresults[p] == MEC_OK && is_whole_algo(r->valgos[p])) counts[whole_group(r->valgos[p])]++;
  for (int g = 0, at = 0; g < kWholeGroups; g++) { first[g] = at; at += static_cast<int>(counts[g]); }
}

// Completes the batch that ran on slot `s` (rc: how its stream ended) and wakes its callers.
static void batcher_finish(mec_batcher* b, InflightBatch& fb, Slot& s, int rc) {
  mec_codec* c = b->codec;
  if (fb.kind == ReqKind::Verify) {
    // the frame verdicts in s.flags.h and the whole-file digests in s.wdig.h, both in batcher_submit_verify's order
    const uint8_t* fl = static_cast<const uint8_t*>(s.flags.h.p);
    const uint8_t* wd = static_cast<const uint8_t*>(s.wdig.h.p);
    const int64_t S = c->S();
    int64_t frame = 0, next[kWholeGroups];
    verify_whole_firsts(fb.reqs, next);
    for (BatchReq* r : fb.reqs) {
      r->result = rc;
      if (rc != MEC_OK) continue;
      for (int64_t p = 0; p < r->vparts; p++) {
        if (r->vresults[p] != MEC_OK) continue;
        const int a = r->valgos[p];
        bool bad = false;
        if (a == MEC_HIGHWAYHASH256S) {
          for (int64_t j = ceil_frac(r->vpart_lens[p], S); j > 0; j--) bad |= fl[frame++] != 0;
        } else {
          const int64_t q = next[whole_group(a)]++;
          bad = memcmp(wd + q * 64, r->vsums + p * 64, static_cast<size_t>(mec_digest_size(a))) != 0;  // cmd/bitrot.go:171-173
        }
        if (bad) r->vresults[p] = MEC_ERR_FILE_CORRUPT;
      }
      b->st_verifies++;
    }
  } else if (is_read(fb.kind)) {
    // per-frame digest verdicts of the merged launch: a request that met a corrupt frame is redone on its own; the others are done
    // (their bytes are in place; a heal's `corrupt` was zeroed when it was queued).  A whole-file reader has no frames: the flags at
    // its arena position mean nothing, and the digest of its staged shard file (batch_whole_stage: streams in request order, a
    // request's in ascending position order, digest j at s.wdig.h + j*64) is compared with its expected sum instead.
    const uint8_t* fl = static_cast<const uint8_t*>(s.flags.h.p);
    const uint8_t* wd = static_cast<const uint8_t*>(s.wdig.h.p);
    const BatchGetDesc* tab = static_cast<const BatchGetDesc*>(s.dreq.h.p);
    const int k = c->k;
    int64_t stream = 0;
    for (size_t q = 0; q < fb.reqs.size(); q++) {
      BatchReq* r = fb.reqs[q];
      int64_t res = rc != MEC_OK ? rc : r->kind == ReqKind::Heal ? MEC_OK : is_move(r->kind) ? r->total : r->sse_key ? r->sse_len : r->length;
      if (rc == MEC_OK) {
        bool bad = false;
        const uint32_t wpos = r->whole_algo ? tab[q].whole_pos : 0;
        if (wpos) {
          const size_t ds = static_cast<size_t>(mec_digest_size(r->whole_algo));
          for (int t = 0; t < k; t++)
            if ((wpos >> t) & 1) bad |= memcmp(wd + stream++ * 64, r->whole_sums + static_cast<size_t>(tab[q].chosen[t]) * 64, ds) != 0;
        }
        for (int64_t bb = 0; bb < r->get_nblocks && !bad; bb++) {
          const int64_t slot = (r->get_tail_slot >= 0 && bb == r->get_nblocks - 1) ? r->get_tail_slot : r->get_slot0 + bb;
          for (int t = 0; t < k; t++) bad |= !((wpos >> t) & 1) && fl[slot * k + t] != 0;
        }
        if (bad) {
          b->st_redone++;
          res = batcher_run_alone(b, *r);
        } else {
          if (r->heal_hint) *r->heal_hint = 0;
          if (r->sse_key) {  // the verdicts of its packages (sse_get_open): a package that fails hands out nothing of the range
            const uint8_t* v = static_cast<const uint8_t*>(s.sse_st.h.p) + r->sse_row0;
            const int64_t nrows = (r->sse_offset + r->sse_len - 1) / kPkg - r->sse_offset / kPkg + 1;
            int64_t e = MEC_OK;
            for (int64_t j = 0; j < nrows; j++) {
              if (v[j] == kDareUnsupported) e = MEC_ERR_UNSUPPORTED;
              else if (v[j] != kDareOk && e == MEC_OK) e = MEC_ERR_NOT_AUTHENTIC;
            }
            if (e != MEC_OK) {
              memset(r->dst, 0, static_cast<size_t>(r->sse_len));
              res = e;
            } else {
              b->st_sse_gets++;
            }
          }
          if (r->kind == ReqKind::Transcode) b->st_transcodes++;
          if (r->kind == ReqKind::TranscodeWhole) b->st_transcodes_whole++;
          if (r->algos && r->whole_algo) b->st_reads_whole++;
        }
      }
      r->result = res;
    }
  } else {
    for (size_t q = 0; q < fb.reqs.size(); q++) {
      BatchReq* r = fb.reqs[q];
      if (rc == MEC_OK && fb.needs_retire) frames_retire(c, r->ch, r->files, r->with_data, r->data_digests);
      if (rc == MEC_OK && r->crc_which) {  // batcher_crc_enqueue's results, row q of the slot's pinned mirror
        const uint64_t* h = static_cast<const uint64_t*>(s.crc_out.h.p) + q * kCrcTypes;
        for (int ty = 0; ty < kCrcTypes; ty++) r->crc_out[ty] = h[ty];
        b->st_crc_requests++;
      }
      if (rc == MEC_OK && r->sum_which) {  // batcher_sums_fork's records, record q of the slot's pinned mirror
        const uint8_t* h = static_cast<const uint8_t*>(s.sum_out.h.p) + q * kSumRecord;
        for (int a = 0; a < kSumAlgos; a++)
          if (r->sum_which & (MEC_SUM_MD5 << a)) memcpy(r->sums + 32 * a, h + 32 * a, static_cast<size_t>(sum_digest_len(a)));
        b->st_sum_requests++;
      }
      if (rc == MEC_OK && r->sse_key) b->st_sse_puts++;
      r->result = rc != MEC_OK ? rc : r->sse_key ? r->sse_len : r->len;
    }
  }
  if (s.sse_heads) {  // the key heads this batch wrote (the device copy was zeroed behind the cipher)
    explicit_bzero(s.hsse_keys.p, static_cast<size_t>(s.sse_heads) * kDareKeyHead);
    s.sse_heads = 0;
  }
  {
    std::lock_guard<std::mutex> lk(b->mu);
    for (BatchReq* r : fb.reqs) { r->done = true; r->cv.notify_one(); }  // under the lock: `r` lives on its caller's stack
  }
  fb.reqs.clear();
}

// With sw.trace, records mark j of the batch on the batcher's slot `s`: 0 before staging, 1 staged, 2 encoded or rebuilt, 3 done
// (mec_batcher_stat "us_stage", "us_kernel" and "us_scatter" sum the gaps)
static void mark_phase(mec_batcher* b, Slot& s, int j) {
  if (b->sw.trace) cudaEventRecord(b->ev_ph[&s - b->codec->slots][j], s.st);
}

// Object checksums of the PUTs of a batch that asked for them (mec_batcher_encode_crc).  Request q's bytes are two segments of s.src,
// its full blocks at ch.d_src and its short last block at ch.d_src_tail; each is cut into kCrcRegion work items.  batcher_crc_table
// writes the work table and enqueues its copy ahead of the staging (behind other slots' staging on the copy engine it would hold up
// this batch's kernels); batcher_crc_launch, enqueued once the batch is staged, runs the region kernel over every item and the fold
// kernel that merges each request's items into row q of s.crc_out, and copies the rows to s.crc_out.h, where batcher_finish reads them.
// Two launches and one small copy each way per batch, whatever the number of requests; a batch without such requests (p->nreq == 0)
// enqueues nothing.  The buffers were sized by mec_batcher_new; they only grow here for a batch led by a request larger than
// max_batch_blocks.
static int batcher_crc_table(mec_batcher* b, Slot& s, const std::vector<BatchReq*>& reqs, CrcSegParams* p) {
  *p = CrcSegParams();
  int which = 0;
  for (BatchReq* r : reqs) which |= r->crc_which;
  if (!which) return MEC_OK;
  mec_codec* c = b->codec;
  const int64_t bs = c->block_size;
  const uint8_t* base = static_cast<const uint8_t*>(s.src.p);
  auto regions = [](int64_t n) { return (n + kCrcRegion - 1) / kCrcRegion; };
  int64_t nwork = 0;
  for (BatchReq* r : reqs)
    if (r->crc_which) nwork += regions(r->ch.nfull * bs) + regions(r->ch.tail);
  const size_t nreq = reqs.size(), tab_bytes = nreq * sizeof(CrcReq) + static_cast<size_t>(nwork) * sizeof(CrcWork);
  int rc;
  if ((rc = s.crc_tab.ensure(tab_bytes))) return rc;
  if ((rc = s.crc_part.ensure(static_cast<size_t>(nwork) * kCrcTypes * sizeof(uint64_t)))) return rc;
  if ((rc = s.crc_out.ensure(nreq * kCrcTypes * sizeof(uint64_t)))) return rc;
  CrcReq* rt = static_cast<CrcReq*>(s.crc_tab.h.p);
  CrcWork* wt = reinterpret_cast<CrcWork*>(rt + nreq);
  int64_t w = 0;
  for (size_t q = 0; q < nreq; q++) {
    const BatchReq* r = reqs[q];
    rt[q] = CrcReq{static_cast<int32_t>(w), 0, r->crc_which, 0};
    if (r->crc_which) {
      auto segment = [&](const uint8_t* p, int64_t n) {
        for (int64_t off = 0; off < n; off += kCrcRegion)
          wt[w++] = CrcWork{(p - base) + off, static_cast<int32_t>(std::min(kCrcRegion, n - off)), r->crc_which};
      };
      segment(r->ch.d_src, r->ch.nfull * bs);
      segment(r->ch.d_src_tail, r->ch.tail);
    }
    rt[q].w1 = static_cast<int32_t>(w);
  }
  MEC_CUDA_OK(s.crc_tab.upload(tab_bytes, s.st));
  p->base = base;
  p->reqs = static_cast<const CrcReq*>(s.crc_tab.d.p);
  p->work = reinterpret_cast<const CrcWork*>(p->reqs + nreq);
  p->nwork = nwork; p->nreq = static_cast<int>(nreq); p->which = which;
  p->tables = static_cast<const CrcTables*>(c->crc_tables.p);
  p->partial = static_cast<uint64_t*>(s.crc_part.p);
  p->out = static_cast<uint64_t*>(s.crc_out.d.p);
  return MEC_OK;
}
static int batcher_crc_launch(mec_batcher* b, Slot& s, const CrcSegParams& p) {
  if (p.nreq == 0) return MEC_OK;
  mec_codec* c = b->codec;
  const unsigned grid = static_cast<unsigned>(std::min<int64_t>(p.nwork, static_cast<int64_t>(c->eng->num_sms()) * 8));
  crc_seg_regions_kernel<<<grid, kCrcThreads, 0, s.st>>>(p);
  MEC_CUDA_OK(cudaGetLastError());
  c->eng->count_launch();
  crc_seg_fold_kernel<<<static_cast<unsigned>(ceil_frac(static_cast<int64_t>(p.nreq) * 32, kCrcFoldThreads)), kCrcFoldThreads, 0, s.st>>>(p);
  MEC_CUDA_OK(cudaGetLastError());
  c->eng->count_launch();
  MEC_CUDA_OK(s.crc_out.download(static_cast<size_t>(p.nreq) * kCrcTypes * sizeof(uint64_t), s.st));
  return MEC_OK;
}

// Object hashes of the PUTs of a batch that asked for them (mec_batcher_encode_sums): one work item per (request, algorithm) over
// the request's two segments of s.src (full blocks at ch.d_src, short last block at ch.d_src_tail), record q of s.sum_out for
// request q.  batcher_sums_table writes the table and enqueues its copy ahead of the staging, as batcher_crc_table does, and
// returns the number of items (0: the batch enqueues nothing for hashes).  batcher_sums_fork, enqueued once the batch is staged,
// runs ONE stream_sums_kernel on the slot's second stream; batcher_sums_join makes the slot's stream wait for it and copies the
// records to s.sum_out.h, where batcher_finish reads them.  The buffers were sized by mec_batcher_new; they only grow here for a batch led
// by a request larger than max_batch_blocks.
static int batcher_sums_table(mec_batcher* b, Slot& s, const std::vector<BatchReq*>& reqs, int64_t* nwork) {
  *nwork = 0;
  for (BatchReq* r : reqs) *nwork += __builtin_popcount(static_cast<unsigned>(r->sum_which));
  if (*nwork == 0) return MEC_OK;
  const int64_t bs = b->codec->block_size;
  const size_t bytes = static_cast<size_t>(*nwork) * sizeof(SumWork);
  int rc;
  if ((rc = s.sum_tab.ensure(bytes))) return rc;
  if ((rc = s.sum_out.ensure(reqs.size() * kSumRecord))) return rc;
  const uint8_t* base = static_cast<const uint8_t*>(s.src.p);
  SumWork* t = static_cast<SumWork*>(s.sum_tab.h.p);
  int64_t w = 0;
  for (size_t q = 0; q < reqs.size(); q++) {
    const EncChunk& ch = reqs[q]->ch;
    w = sum_items(t, w, reqs[q]->sum_which, static_cast<int64_t>(q) * kSumRecord, ch.nfull ? ch.d_src - base : 0, ch.nfull * bs,
                  ch.tail ? ch.d_src_tail - base : 0, ch.tail);
  }
  sum_sort(t, w);
  MEC_CUDA_OK(s.sum_tab.upload(bytes, s.st));
  return MEC_OK;
}
static int batcher_sums_fork(mec_batcher* b, Slot& s, int64_t nwork) {
  if (nwork == 0) return MEC_OK;
  const int si = static_cast<int>(&s - b->codec->slots);
  MEC_CUDA_OK(cudaEventRecord(b->ev_staged[si], s.st));
  MEC_CUDA_OK(cudaStreamWaitEvent(b->sum_st[si], b->ev_staged[si], 0));
  int rc = sum_launch(b->codec, static_cast<const uint8_t*>(s.src.p), static_cast<const SumWork*>(s.sum_tab.d.p), nwork,
                      static_cast<uint8_t*>(s.sum_out.d.p), b->sum_st[si]);
  if (rc) return rc;
  MEC_CUDA_OK(cudaEventRecord(b->ev_summed[si], b->sum_st[si]));
  return MEC_OK;
}
static int batcher_sums_join(mec_batcher* b, Slot& s, size_t nreq, int64_t nwork) {
  if (nwork == 0) return MEC_OK;
  MEC_CUDA_OK(cudaStreamWaitEvent(s.st, b->ev_summed[&s - b->codec->slots], 0));
  MEC_CUDA_OK(s.sum_out.download(nreq * kSumRecord, s.st));
  return MEC_OK;
}

// Server-side encryption in merged batches (mec_batcher_encode_sse / _decode_sse).  The encrypted requests of a batch are the streams
// of ONE dare_setup_kernel launch (stream z = the z-th such request in batch order) and their packages the rows of ONE dare_kernel
// launch.  Each request carries the option "dare_chacha20" it was admitted with: an open batch with a request at 1 or 2 adds ONE
// dare_chacha_kernel launch behind the AES one (each stream's key head says whether it opens ChaCha20); a seal batch seals the
// packages of its requests at 2 with ONE dare_chacha_kernel launch instead, and needs the setup only for the others.  Each slot
// has its own key table, package table (s.dpk) and verdicts: six batches in flight never share key material.  The device keys are
// zeroed on the slot's stream behind the cipher launches, the host-written heads by batcher_finish.
static int sse_batch_setup(mec_batcher* b, Slot& s, const std::vector<BatchReq*>& reqs, bool seal, int64_t* nsse) {
  *nsse = 0;
  bool aes = !seal;
  for (const BatchReq* r : reqs)
    if (r->sse_key) { ++*nsse; aes |= r->sse_chacha != 2; }
  if (*nsse == 0) return MEC_OK;
  int rc;
  if ((rc = s.sse_keys.ensure(static_cast<size_t>(*nsse) * sizeof(DareStreamKeys))) ||
      (rc = s.hsse_keys.ensure(static_cast<size_t>(*nsse) * kDareKeyHead)))
    return rc;
  uint8_t* h = static_cast<uint8_t*>(s.hsse_keys.p);
  for (const BatchReq* r : reqs)
    if (r->sse_key) { dare_key_head(h, r->sse_key, seal ? r->sse_nonce : nullptr, r->sse_chacha); h += kDareKeyHead; }
  s.sse_heads = *nsse;
  return dare_setup(b->codec, static_cast<DareStreamKeys*>(s.sse_keys.p), static_cast<const uint8_t*>(s.hsse_keys.p), *nsse, s.st, aes);
}
// The plaintext arena: sized for a full batch (batcher_slot_blocks x block_size) on the slot's first encrypted batch; it only grows
// past that for a batch led by a request larger than max_batch_blocks.  A batch's plaintext is at most its ciphertext, which batch
// formation bounds.
static int64_t batcher_slot_blocks(const mec_batcher* b);
static int size_sse_arena(mec_batcher* b, Slot& s, int64_t bytes) {
  return s.sse_pt.ensure(static_cast<size_t>(std::max(bytes, batcher_slot_blocks(b) * b->codec->block_size)));
}
// The cipher launches over the batch's package rows s.dpk.h[0, rows) (an open writes its verdicts to s.sse_st), then the keys are
// zeroed.  A seal seals rows [0, chacha_from) with AES-256-GCM and the rest with ChaCha20-Poly1305; an open with chacha_from < rows
// adds the ChaCha20 open behind the AES one.
static int sse_batch_cipher(mec_batcher* b, Slot& s, bool seal, int64_t nsse, int64_t rows, int64_t chacha_from, const uint8_t* in,
                            uint8_t* out) {
  MEC_CUDA_OK(s.dpk.upload(static_cast<size_t>(rows) * sizeof(DarePkg), s.st));
  const DareStreamKeys* k = static_cast<const DareStreamKeys*>(s.sse_keys.p);
  const DarePkg* pk = static_cast<const DarePkg*>(s.dpk.d.p);
  int rc;
  if (seal) {
    if ((rc = dare_launch(b->codec, true, false, k, pk, chacha_from, in, out, nullptr, s.st)) ||
        (rc = dare_launch(b->codec, true, true, k, pk + chacha_from, rows - chacha_from, in, out, nullptr, s.st)))
      return rc;
  } else if ((rc = dare_launch(b->codec, false, chacha_from < rows, k, pk, rows, in, out, static_cast<uint8_t*>(s.sse_st.d.p), s.st))) {
    return rc;
  }
  MEC_CUDA_OK(cudaMemsetAsync(s.sse_keys.p, 0, static_cast<size_t>(nsse) * sizeof(DareStreamKeys), s.st));
  return MEC_OK;
}

// The encrypted PUTs of a batch, before its staging copy: their plaintext goes to the arena s.sse_pt by pieces added to `h2d` (the
// batch's one batched copy), their packages are laid out contiguously per request in the ciphertext arena s.aux (unused by PUT
// batches; r->sse_ct), and the key setup is enqueued.  *rows = 0: the batch has no encrypted request.  The rows of the requests
// admitted at option 2 (ChaCha20-Poly1305) come last, from *chacha_from on.
static int sse_put_plan(mec_batcher* b, Slot& s, const std::vector<BatchReq*>& reqs, CopyList& h2d, int64_t* nsse, int64_t* rows,
                        int64_t* chacha_from) {
  *rows = 0;
  int64_t pt_total = 0, ct_total = 0;
  for (const BatchReq* r : reqs)
    if (r->sse_key) {
      *rows += ceil_frac(r->sse_len, kPkg);
      pt_total += round_up(r->sse_len, 256);
      ct_total += round_up(r->len, 256);
    }
  if (*rows == 0) return MEC_OK;
  int rc;
  if ((rc = size_sse_arena(b, s, pt_total)) || (rc = s.aux.ensure(static_cast<size_t>(ct_total))) ||
      (rc = s.dpk.ensure(static_cast<size_t>(*rows) * sizeof(DarePkg))))
    return rc;
  DarePkg* t = static_cast<DarePkg*>(s.dpk.h.p);
  uint8_t* pt = static_cast<uint8_t*>(s.sse_pt.p);
  int64_t w = 0, po = 0, co = 0;
  for (int pass = 0; pass < 2; pass++) {  // the AES-256-GCM requests, then the ChaCha20-Poly1305 ones
    if (pass == 1) *chacha_from = w;
    int z = 0;  // the request's stream: its place among the batch's encrypted requests
    for (BatchReq* r : reqs) {
      if (!r->sse_key) continue;
      if ((r->sse_chacha == 2) != (pass == 1)) { z++; continue; }
      const int64_t np = ceil_frac(r->sse_len, kPkg);
      for (int64_t j = 0; j < np; j++) t[w++] = dare_row(po + j * kPkg, co + j * kEPkg, 0, std::min(kPkg, r->sse_len - j * kPkg), j, z, j == np - 1);
      h2d.add(pt + po, r->src, r->sse_len);
      r->sse_ct = co;
      po += round_up(r->sse_len, 256);
      co += round_up(r->len, 256);
      z++;
    }
  }
  return sse_batch_setup(b, s, reqs, true, nsse);
}
// Once the batch is staged: ONE seal launch over every package (each sealed once), then ONE batched device-to-device copy of each
// request's ciphertext into its places in the PUT layout (full blocks at ch.d_src, the short last block at ch.d_src_tail)
static int sse_put_seal(mec_batcher* b, Slot& s, const std::vector<BatchReq*>& reqs, int64_t nsse, int64_t rows, int64_t chacha_from) {
  if (rows == 0) return MEC_OK;
  const uint8_t* ct = static_cast<const uint8_t*>(s.aux.p);
  int rc = sse_batch_cipher(b, s, true, nsse, rows, chacha_from, static_cast<const uint8_t*>(s.sse_pt.p), static_cast<uint8_t*>(s.aux.p));
  if (rc) return rc;
  const int64_t bs = b->codec->block_size;
  CopyList cl;
  for (const BatchReq* r : reqs) {
    if (!r->sse_key) continue;
    cl.add(const_cast<uint8_t*>(r->ch.d_src), ct + r->sse_ct, r->ch.nfull * bs);
    cl.add(const_cast<uint8_t*>(r->ch.d_src_tail), ct + r->sse_ct + r->ch.nfull * bs, r->ch.tail);
  }
  return cl.flush(s.st);
}

// The encrypted GETs of a batch, once the scatter has put each one's ciphertext range (whole packages) at s.src + asm_off[q]: ONE
// setup and ONE open launch over every package into the arena s.sse_pt, the verdicts back to s.sse_st.h (r->sse_row0 on), and ONE
// batched copy of each request's plaintext range to its caller.  The arena is cleared first, so a package that fails leaves zeros.
static int sse_get_open(mec_batcher* b, Slot& s, const std::vector<BatchReq*>& reqs, const std::vector<int64_t>& asm_off) {
  int64_t rows = 0, pt_total = 0;
  bool chacha = false;
  for (const BatchReq* r : reqs)
    if (r->sse_key) {
      const int64_t np = (r->sse_offset + r->sse_len - 1) / kPkg - r->sse_offset / kPkg + 1;
      rows += np;
      pt_total += np * kPkg;
      chacha |= r->sse_chacha >= 1;
    }
  if (rows == 0) return MEC_OK;
  int rc;
  if ((rc = size_sse_arena(b, s, pt_total)) || (rc = s.dpk.ensure(static_cast<size_t>(rows) * sizeof(DarePkg))) || (rc = s.sse_st.ensure(static_cast<size_t>(rows))))
    return rc;
  int64_t nsse;
  if ((rc = sse_batch_setup(b, s, reqs, false, &nsse))) return rc;
  DarePkg* t = static_cast<DarePkg*>(s.dpk.h.p);
  uint8_t* pt = static_cast<uint8_t*>(s.sse_pt.p);
  CopyList d2h;
  int64_t w = 0, po = 0;
  int z = 0;
  for (size_t q = 0; q < reqs.size(); q++) {
    BatchReq* r = reqs[q];
    if (!r->sse_key) continue;
    const int64_t D = r->sse_total, npk = ceil_frac(D, kPkg);
    const int64_t p0 = r->sse_offset / kPkg, np = (r->sse_offset + r->sse_len - 1) / kPkg - p0 + 1;
    r->sse_row0 = w;
    for (int64_t j = 0; j < np; j++) {
      const int64_t p = p0 + j;
      t[w++] = dare_row(asm_off[q] + j * kEPkg, po + j * kPkg, asm_off[q], p == npk - 1 ? D - p * kPkg : kPkg, p, z, p == npk - 1);
    }
    d2h.add(r->dst, pt + po + (r->sse_offset - p0 * kPkg), r->sse_len);
    b->codec->st_d2h += r->sse_len;
    po += np * kPkg;
    z++;
  }
  MEC_CUDA_OK(cudaMemsetAsync(pt, 0, static_cast<size_t>(pt_total), s.st));
  if ((rc = sse_batch_cipher(b, s, false, nsse, rows, chacha ? 0 : rows, static_cast<const uint8_t*>(s.src.p), pt))) return rc;
  MEC_CUDA_OK(s.sse_st.download(static_cast<size_t>(rows), s.st));
  return d2h.flush(s.st);
}

// The PUT layout of a merged batch on slot `s` of codec `c`, in request order: every request's full blocks contiguous from s.src
// (from block full0 on), the short last blocks behind all of them at 256-byte-rounded offsets (block tail_slot, byte tail_src_off);
// parity rows [block][m][pitch] in s.out, digests [block][n][32] in s.dig.  A request is r->len object bytes for the frames in
// r->files.  Sizes those buffers and fills request q's row of the BatchReqDesc table in s.dreq.h (`rows`) and / or its EncChunk
// r->ch, whose digests come back to s.dig.h (`chunks`).
struct PutLayout {
  int64_t total_full = 0, nslots = 0, max_nb = 0;  // full blocks, all blocks, the most blocks of one request
};
static int put_layout(mec_codec* c, Slot& s, const std::vector<BatchReq*>& reqs, bool rows, bool chunks, PutLayout& lay) {
  const int m = c->m, n = c->n;
  const int64_t bs = c->block_size, pitch = round_up(c->S(), 16);
  int64_t ntails = 0, tail_bytes = 0;
  for (const BatchReq* r : reqs) {
    lay.total_full += r->len / bs;
    if (r->len % bs) { ntails++; tail_bytes += round_up(r->len % bs, 256); }
  }
  lay.nslots = lay.total_full + ntails;
  const int64_t nb1 = std::max<int64_t>(lay.nslots, 1);
  int rc;
  if ((rc = s.src.ensure(static_cast<size_t>(lay.total_full * bs + tail_bytes + 512)))) return rc;
  if ((rc = s.out.ensure(static_cast<size_t>(nb1 * std::max(m, 1) * pitch)))) return rc;
  if ((rc = s.dig.d.ensure(static_cast<size_t>(nb1 * n * 32)))) return rc;
  if (chunks && (rc = s.dig.h.ensure(static_cast<size_t>(nb1 * n * 32)))) return rc;
  if (rows && (rc = s.dreq.ensure(reqs.size() * sizeof(BatchReqDesc)))) return rc;
  uint8_t* dsrc = static_cast<uint8_t*>(s.src.p);
  uint8_t* dout = static_cast<uint8_t*>(s.out.p);
  const uint8_t* hdig = static_cast<const uint8_t*>(s.dig.h.p);
  BatchReqDesc* tab = static_cast<BatchReqDesc*>(s.dreq.h.p);
  int64_t fb = 0, tb = lay.total_full, toff = lay.total_full * bs;
  for (size_t q = 0; q < reqs.size(); q++) {
    BatchReq* r = reqs[q];
    const int64_t nf = r->len / bs, tl = r->len % bs;
    if (rows) {
      BatchReqDesc& d = tab[q];
      memset(&d, 0, sizeof(d));
      d.src = r->src; d.len = r->len; d.data_digests = r->data_digests; d.with_data = r->with_data ? 1 : 0;
      for (int i = 0; i < n; i++) d.files[i] = r->files[i];
      d.full0 = fb; d.tail_slot = tl ? tb : -1; d.tail_src_off = tl ? toff : 0;
    }
    if (chunks) {
      EncChunk& ch = r->ch;
      ch = EncChunk();
      ch.nfull = nf; ch.tail = tl; ch.nb = nf + (tl ? 1 : 0);
      ch.s = &s; ch.st = s.st; ch.pitch = pitch;
      ch.d_src = dsrc + fb * bs; ch.d_out = dout + fb * m * pitch; ch.h_dig = hdig + fb * n * 32;
      if (tl) { ch.d_src_tail = dsrc + toff; ch.d_out_tail = dout + tb * m * pitch; ch.h_dig_tail = hdig + tb * n * 32; }
    }
    fb += nf;
    if (tl) { tb++; toff += round_up(tl, 256); }
    lay.max_nb = std::max(lay.max_nb, nf + (tl ? 1 : 0));
  }
  return MEC_OK;
}

// Encode and frame scatter of a staged batch in the PUT layout (`tab`, `lay`: put_layout; `cp` describes the staging): ONE latency
// launch with a per-block geometry table when the batch fits one, otherwise one launch over all full blocks plus one per short
// block; then the scatter kernel writes every frame into every caller's part-file images.  Used by merged PUTs on the batcher's
// codec and by merged transcodes on the destination codec (slot `s` of codec `c`, enqueued on stream `st`).  `ev_encoded` (may be
// null) is recorded between the encode and the scatter.
static int batch_encode_scatter(mec_codec* c, Slot& s, cudaStream_t st, const BatchReqDesc* tab, size_t nreq, const PutLayout& lay,
                                const BatchCopyParams& cp, cudaEvent_t ev_encoded) {
  const int k = c->k, m = c->m, n = c->n;
  const int64_t bs = c->block_size, S = c->S(), pitch = round_up(S, 16);
  const int64_t total_full = lay.total_full, nslots = lay.nslots;
  uint8_t* dsrc = static_cast<uint8_t*>(s.src.p);
  uint8_t* dout = static_cast<uint8_t*>(s.out.p);
  uint8_t* ddig = static_cast<uint8_t*>(s.dig.d.p);
  int rc;
  if (c->eng->small_ok(c->opt, nslots)) {
    // ONE launch for every block of the batch, full or short (objects smaller than a block are nothing but a short block): the
    // latency kernel takes the geometry of each block from a table
    if ((rc = s.blk.ensure(static_cast<size_t>(nslots) * sizeof(SmallBlock)))) return rc;
    SmallBlock* bt = static_cast<SmallBlock*>(s.blk.h.p);
    for (int64_t q = 0; q < total_full; q++) bt[q] = SmallBlock{q * bs, static_cast<int32_t>(S), static_cast<int32_t>(bs)};
    for (size_t q = 0; q < nreq; q++)
      if (tab[q].tail_slot >= 0) {
        const int64_t tl = tab[q].len % bs;
        bt[tab[q].tail_slot] = SmallBlock{tab[q].tail_src_off, static_cast<int32_t>(ceil_frac(tl, k)), static_cast<int32_t>(tl)};
      }
    MEC_CUDA_OK(s.blk.upload(static_cast<size_t>(nslots) * sizeof(SmallBlock), st));
    FusedDesc d;
    d.k = k; d.r = m;
    d.coef = c->matrix.data() + static_cast<size_t>(k) * k;
    d.static_encode = true; d.contiguous = true; d.key = kMagicKey; d.out_pitch = pitch;
    d.nblocks = nslots; d.S = static_cast<int32_t>(S);
    d.in_base = dsrc; d.in_block_stride = bs; d.in_block_len = bs;
    d.out = dout; d.digests = ddig;
    d.blocks = static_cast<const SmallBlock*>(s.blk.d.p);
    if ((rc = c->eng->launch_fused(d, c->opt, st))) return rc;
  } else {
    if (total_full > 0 && (rc = encode_device_locked(c, dsrc, total_full * bs, dout, pitch, ddig, st))) return rc;
    for (size_t q = 0; q < nreq; q++)
      if (tab[q].tail_slot >= 0 &&
          (rc = encode_device_locked(c, dsrc + tab[q].tail_src_off, tab[q].len % bs, dout + tab[q].tail_slot * m * pitch, pitch,
                                     ddig + tab[q].tail_slot * n * 32, st)))
        return rc;
  }
  if (ev_encoded) cudaEventRecord(ev_encoded, st);
  batch_scatter_kernel<<<dim3(static_cast<unsigned>(std::min<int64_t>(lay.max_nb, 16)), static_cast<unsigned>(n), static_cast<unsigned>(nreq)), 128, 0, st>>>(cp);
  MEC_CUDA_OK(cudaGetLastError());
  c->eng->count_launch();
  return MEC_OK;
}

// stage, launch and enqueue the copy-back of one merged batch on slot `s`; *nblocks = the erasure blocks it encodes
static int batcher_submit(mec_batcher* b, Slot& s, std::vector<BatchReq*>& reqs, bool* needs_retire, int64_t* nblocks) {
  mec_codec* c = b->codec;
  const int k = c->k, m = c->m, n = c->n;
  const int64_t bs = c->block_size, S = c->S(), pitch = round_up(S, 16);
  *needs_retire = true;
  bool all_mapped = n <= kBatchMaxFiles && !b->sw.memcpy, sse = false;
  for (BatchReq* r : reqs) { all_mapped &= r->mapped; sse |= r->sse_key != nullptr; }
  int64_t nsse = 0, sse_rows = 0, sse_chacha_from = 0;
  PutLayout lay;
  int rc;
  if ((rc = put_layout(c, s, reqs, all_mapped, true, lay))) return rc;
  const int64_t nslots = lay.nslots;
  *nblocks = nslots;
  uint8_t* dsrc = static_cast<uint8_t*>(s.src.p);
  uint8_t* dout = static_cast<uint8_t*>(s.out.p);
  uint8_t* ddig = static_cast<uint8_t*>(s.dig.d.p);
  if (all_mapped) {
    // gather kernel -> ONE fused launch over all full blocks (+ one per tail) -> scatter kernel: a handful of launches and one
    // small table copy per batch, whatever the number of requests
    const BatchReqDesc* tab = static_cast<const BatchReqDesc*>(s.dreq.h.p);
    for (const BatchReq* r : reqs) {
      const int64_t nf = r->len / bs, tl = r->len % bs;
      c->st_h2d += r->sse_key ? r->sse_len : r->len;
      c->st_d2h += (nf * S + (tl ? ceil_frac(tl, k) : 0)) * (r->with_data ? n : m);
    }
    const int si = static_cast<int>(&s - c->slots);
    mark_phase(b, s, 0);
    MEC_CUDA_OK(s.dreq.upload(reqs.size() * sizeof(BatchReqDesc), s.st));
    CrcSegParams crc;
    if ((rc = batcher_crc_table(b, s, reqs, &crc))) return rc;
    int64_t nsum;
    if ((rc = batcher_sums_table(b, s, reqs, &nsum))) return rc;
    BatchCopyParams cp;
    cp.reqs = static_cast<const BatchReqDesc*>(s.dreq.d.p);
    cp.nreq = static_cast<int>(reqs.size()); cp.k = k; cp.m = m; cp.bs = bs; cp.S = S; cp.pitch = pitch;
    cp.staged = dsrc; cp.parity = dout; cp.digests = ddig;
    // staging: the copy engines are the faster reader of host memory (one call per request); the gather kernel (SM loads over
    // PCIe, no per-request call at all) is kept for hosts where the worker thread is the bottleneck
    // requests [0, ndma) go through the copy engine, [ndma, nreq) through the gather kernel on the aux stream, concurrently
    // (a batch with encrypted requests stages all of them by the copy engine: their plaintext goes to the arena, not the layout)
    size_t ndma = b->sw.gather && !sse ? 0 : reqs.size();
    if (!b->sw.gather && !sse && b->sw.gather_pct > 0 && b->aux && reqs.size() >= 8)
      ndma = reqs.size() - reqs.size() * static_cast<size_t>(b->sw.gather_pct) / 100;
    if (ndma < reqs.size()) {
      cudaStream_t gs = s.st;
      if (ndma > 0) {
        gs = b->aux;
        MEC_CUDA_OK(cudaEventRecord(b->ev_table[si], s.st));
        MEC_CUDA_OK(cudaStreamWaitEvent(gs, b->ev_table[si], 0));
      }
      int64_t glen = 0;
      for (size_t q = ndma; q < reqs.size(); q++) glen = std::max(glen, tab[q].len);
      BatchCopyParams gp = cp;
      gp.reqs = cp.reqs + ndma;
      gp.nreq = static_cast<int>(reqs.size() - ndma);
      const unsigned gx = static_cast<unsigned>(std::min<int64_t>(64, std::max<int64_t>(1, ceil_frac(glen, 32 << 10))));
      batch_gather_kernel<<<dim3(gx, static_cast<unsigned>(gp.nreq)), 256, 0, gs>>>(gp);
      MEC_CUDA_OK(cudaGetLastError());
      c->eng->count_launch();
      if (ndma > 0) MEC_CUDA_OK(cudaEventRecord(b->ev_gather[si], gs));
    }
    {
      // ONE cudaMemcpyBatchAsync for the whole batch: the copy engine runs a train of 1 MiB pieces at the link rate, faster than the
      // same pieces as separate cudaMemcpyAsync calls (tools/copy_probe.cu compares the two)
      CopyList cl;
      for (size_t q = 0; q < ndma; q++) {
        if (reqs[q]->sse_key) continue;
        const BatchReqDesc& d = tab[q];
        const int64_t fbytes = d.len / bs * bs, tl = d.len - fbytes;
        cl.add(dsrc + d.full0 * bs, d.src, fbytes);
        cl.add(dsrc + d.tail_src_off, d.src + fbytes, tl);
      }
      if ((rc = sse_put_plan(b, s, reqs, cl, &nsse, &sse_rows, &sse_chacha_from))) return rc;
      if ((rc = cl.flush(s.st))) return rc;
    }
    if (ndma > 0 && ndma < reqs.size()) MEC_CUDA_OK(cudaStreamWaitEvent(s.st, b->ev_gather[si], 0));
    if ((rc = sse_put_seal(b, s, reqs, nsse, sse_rows, sse_chacha_from))) return rc;
    mark_phase(b, s, 1);
    if ((rc = batcher_sums_fork(b, s, nsum))) return rc;
    if ((rc = batcher_crc_launch(b, s, crc))) return rc;
    if ((rc = batch_encode_scatter(c, s, s.st, tab, reqs.size(), lay, cp, b->sw.trace ? cudaEvent_t{b->ev_ph[si][2]} : nullptr))) return rc;
    mark_phase(b, s, 3);
    if ((rc = batcher_sums_join(b, s, reqs.size(), nsum))) return rc;
    *needs_retire = false;
    c->st_blocks_encoded += nslots;
    return MEC_OK;
  }
  CrcSegParams crc;
  if ((rc = batcher_crc_table(b, s, reqs, &crc))) return rc;
  int64_t nsum;
  if ((rc = batcher_sums_table(b, s, reqs, &nsum))) return rc;
  for (BatchReq* r : reqs) {
    if (r->sse_key) continue;
    const EncChunk& ch = r->ch;
    if (ch.nfull > 0)
      MEC_CUDA_OK(cudaMemcpyAsync(const_cast<uint8_t*>(ch.d_src), r->src, static_cast<size_t>(ch.nfull * bs), cudaMemcpyHostToDevice, s.st));
    if (ch.tail > 0)
      MEC_CUDA_OK(cudaMemcpyAsync(const_cast<uint8_t*>(ch.d_src_tail), r->src + ch.nfull * bs, static_cast<size_t>(ch.tail), cudaMemcpyHostToDevice, s.st));
    c->st_h2d += r->len;
  }
  if (sse) {  // encrypted requests beside a pageable one: their plaintext in one batched copy, then the seal into the layout
    CopyList cl;
    if ((rc = sse_put_plan(b, s, reqs, cl, &nsse, &sse_rows, &sse_chacha_from)) || (rc = cl.flush(s.st)) ||
        (rc = sse_put_seal(b, s, reqs, nsse, sse_rows, sse_chacha_from)))
      return rc;
    for (const BatchReq* r : reqs) c->st_h2d += r->sse_key ? r->sse_len : 0;
  }
  if ((rc = batcher_sums_fork(b, s, nsum))) return rc;
  if ((rc = batcher_crc_launch(b, s, crc))) return rc;
  if (lay.total_full > 0 && (rc = encode_device_locked(c, dsrc, lay.total_full * bs, dout, pitch, ddig, s.st))) return rc;  // ONE launch for every caller's full blocks
  const uint8_t* hdig = static_cast<const uint8_t*>(s.dig.h.p);
  for (BatchReq* r : reqs) {
    const EncChunk& ch = r->ch;
    if (ch.tail > 0 && (rc = encode_device_locked(c, ch.d_src_tail, ch.tail, ch.d_out_tail, pitch,
                                                  ddig + (ch.h_dig_tail - hdig), s.st)))
      return rc;
  }
  MEC_CUDA_OK(s.dig.download(static_cast<size_t>(nslots * n * 32), s.st));
  for (BatchReq* r : reqs)
    if ((rc = frames_enqueue(c, r->ch, r->files, r->with_data, r->data_digests))) return rc;
  if ((rc = batcher_sums_join(b, s, reqs.size(), nsum))) return rc;
  c->st_blocks_encoded += nslots;
  return MEC_OK;
}

// Merged GET and heal batches share their plan, layout and staging.  Layout: every request's full blocks first, the short last
// blocks behind them.
struct ReadLayout {
  int64_t nfull_slots = 0, ntails = 0, max_nb = 0;
  size_t table_bytes = 0;  // of the request table (s.dreq.h -> s.dreq)
  int npat = 0;            // distinct erasure patterns of the batch
  const uint8_t* rows = nullptr;  // npat == 1: the r x k decode rows of that pattern
  size_t pat_off = 0, bp_off = 0; // npat > 1: SmallPattern[npat] and the uint16_t pattern of every slot, offsets in the table
  int64_t nslots() const { return nfull_slots + ntails; }
};
// Every request's reader set — the first k readers of its alive mask — and the decode plan of what it rebuilds: the data shards
// those readers miss for a GET, the stale drives for a heal (disjoint from the readers: mec_batcher_heal sends the rest to the
// serial handle).  Fills the request table in s.dreq.h — a heal's carries out_files[targets[q]] of request z at [z * gp.r + q] behind
// the rows; a batch of several patterns then the pattern table and the per-slot pattern index — each request's placement in the
// batch, and gp (gp.r = the most targets of any request).
static int batch_read_plan(mec_batcher* b, Slot& s, std::vector<BatchReq*>& reqs, BatchGetParams& gp, ReadLayout& lay) {
  mec_codec* c = b->codec;
  const int k = c->k, n = c->n;
  const int64_t bs = c->block_size, S = c->S();
  const bool heal = reqs.front()->kind == ReqKind::Heal;
  const size_t nreq = reqs.size();
  if (b->patterns.size() + nreq > kMaxCachedPatterns) b->patterns.clear();  // pointers into the cache stay valid for this batch
  std::vector<const BatchPattern*> pats;
  std::vector<uint64_t> pat_keys;
  std::vector<int> req_pat(nreq);
  std::vector<ReadRange> rrs(nreq);
  int rmax = 0;
  int64_t nslots = 0;
  for (size_t q = 0; q < nreq; q++) {
    const BatchReq* rq = reqs[q];
    uint64_t rmask = 0;
    for (int i = 0, cnt = 0; i < n && cnt < k; i++)
      if ((rq->alive_mask >> i) & 1) { rmask |= 1ull << i; cnt++; }
    const uint64_t tmask = heal ? rq->stale_mask : (~rmask & ((1ull << k) - 1));
    const uint64_t key = rmask | (tmask << 32);  // n <= kBatchMaxFiles = 32
    int pi = 0;
    while (pi < static_cast<int>(pats.size()) && pat_keys[pi] != key) pi++;
    if (pi == static_cast<int>(pats.size())) {
      auto it = b->patterns.find(key);
      if (it == b->patterns.end()) {
        BatchPattern bp;
        int chosen[kMaxShards], nch = 0;
        uint8_t want[kMaxShards] = {};
        for (int i = 0; i < n; i++) {
          if ((rmask >> i) & 1) chosen[nch++] = i;
          want[i] = (tmask >> i) & 1;
        }
        int rc = plan_decode(c, chosen, nch, want, 0, &bp.plan);
        if (rc) return rc;
        memset(&bp.sp, 0, sizeof(bp.sp));
        bp.sp.r = bp.plan.r;
        for (int j = 0; j < bp.plan.r; j++)
          for (int t = 0; t < k; t++) bp.sp.coef[j][t] = bp.plan.rows[static_cast<size_t>(j) * k + t];
        it = b->patterns.emplace(key, std::move(bp)).first;
      }
      pats.push_back(&it->second);
      pat_keys.push_back(key);
      rmax = std::max(rmax, it->second.plan.r);
    }
    req_pat[q] = pi;
    rrs[q] = read_range(c, rq->offset, rq->length, rq->total);
    nslots += rrs[q].nblocks;
  }
  lay.npat = static_cast<int>(pats.size());
  lay.rows = lay.npat == 1 ? pats[0]->plan.rows.data() : nullptr;
  lay.table_bytes = nreq * sizeof(BatchGetDesc) + (heal ? nreq * std::max(rmax, 1) * sizeof(uint8_t*) : 0);
  if (lay.npat > 1) {
    lay.pat_off = round_up(static_cast<int64_t>(lay.table_bytes), 16);
    lay.bp_off = lay.pat_off + pats.size() * sizeof(SmallPattern);
    lay.table_bytes = lay.bp_off + static_cast<size_t>(nslots) * sizeof(uint16_t);
  }
  int rc;
  if ((rc = s.dreq.ensure(lay.table_bytes))) return rc;
  BatchGetDesc* tab = static_cast<BatchGetDesc*>(s.dreq.h.p);
  for (size_t q = 0; q < nreq; q++) {
    BatchReq* rq = reqs[q];
    BatchGetDesc& d = tab[q];
    memset(&d, 0, sizeof(d));
    const ReadRange& rr = rrs[q];
    d.offset = rq->offset; d.length = rq->length; d.total = rq->total; d.dst = rq->dst;
    for (int i = 0; i < n; i++) d.files[i] = rq->gfiles[i];
    d.start_block = rr.start_block; d.nblocks = rr.nblocks;
    d.last_len = rr.last_len;
    const DecodePlan& pl = pats[req_pat[q]]->plan;
    for (int i = 0, t = 0; i < n; i++)
      if (pl.present[i]) d.chosen[t++] = static_cast<int8_t>(i);
    for (int j = 0; j < pl.r; j++) d.targets[j] = static_cast<int8_t>(pl.targets[j]);
    d.r = pl.r;
    d.pattern = req_pat[q];
    for (int t = 0; t < k; t++)
      if ((rq->whole_drives >> d.chosen[t]) & 1) d.whole_pos |= 1u << t;
    const bool tail = rr.last_len != S;
    d.slot0 = lay.nfull_slots;
    lay.nfull_slots += d.nblocks - (tail ? 1 : 0);
    d.tail_slot = tail ? lay.ntails : -1;  // provisional: offset by the number of full slots below
    if (tail) lay.ntails++;
    lay.max_nb = std::max(lay.max_nb, d.nblocks);
    rq->get_nblocks = d.nblocks;
  }
  for (size_t q = 0; q < nreq; q++) {
    tab[q].dma = tab[q].nblocks >= b->sw.dma_blocks ? 1 : 0;
    if (tab[q].tail_slot >= 0) tab[q].tail_slot += lay.nfull_slots;
    reqs[q]->get_slot0 = tab[q].slot0;
    reqs[q]->get_tail_slot = tab[q].tail_slot;
  }
  if (heal) {
    uint8_t** outs = reinterpret_cast<uint8_t**>(tab + nreq);
    for (size_t z = 0; z < nreq; z++)
      for (int q = 0; q < tab[z].r; q++) outs[z * rmax + q] = reqs[z]->outs[tab[z].targets[q]];
  }
  if (lay.npat > 1) {
    uint8_t* base = static_cast<uint8_t*>(s.dreq.h.p);
    SmallPattern* sp = reinterpret_cast<SmallPattern*>(base + lay.pat_off);
    for (int pi = 0; pi < lay.npat; pi++) sp[pi] = pats[pi]->sp;
    uint16_t* bp = reinterpret_cast<uint16_t*>(base + lay.bp_off);
    for (size_t q = 0; q < nreq; q++)
      for (int64_t bb = 0; bb < tab[q].nblocks; bb++) bp[get_slot(tab[q], bb)] = static_cast<uint16_t>(req_pat[q]);
  }
  memset(&gp, 0, sizeof(gp));
  gp.reqs = static_cast<const BatchGetDesc*>(s.dreq.d.p);
  gp.nreq = static_cast<int>(nreq); gp.k = k; gp.r = rmax;
  gp.bs = bs; gp.S = S; gp.P = round_up(32 + S, 16); gp.pitch = round_up(S, 16);
  return MEC_OK;
}

// The raw shard files of the whole-file readers of a merged batch, staged and hashed by batch_whole_stage: position t of request z
// (bit t of its whole_pos) at files + streams[first[z] + whole-file positions of z below t].off on the device.  raw: no request
// of the batch has a streaming reader and no digest is wanted (a GET or move batch), so the reconstruct neither hashes nor verifies.
struct WholeFiles {
  const uint8_t* files;
  const WholeStream* streams;
  const int32_t* first;
  bool raw;
};
static int batch_whole_stage(mec_batcher* b, Slot& s, const std::vector<BatchReq*>& reqs, const BatchGetDesc* tab, WholeFiles* wf);

// The request table to the device, survivor frames of every block of every request -> the slot's arena, the fused reconstruct of
// every request's targets over all of them, and the per-frame digest verdicts back to s.flags.h.  `tab` is the host copy of the table
// gp.reqs points at; gp holds the geometry and gets the arena and rebuilt rows here.  A batch of several erasure patterns is ONE
// latency launch with a decode plan per block (batcher_main only merges such a batch when its blocks fit one).  `wf` (a batch with
// whole-file readers, staged and hashed by batch_whole_stage): their positions are filled from the staged raw shard files by
// batch_whole_rows_kernel, the frame staging skips them, and their verdict flags mean nothing (batcher_finish checks their file
// digests instead).  wf->raw: the reconstruct neither hashes nor verifies anything.
static int batch_read_reconstruct(mec_batcher* b, Slot& s, const BatchGetDesc* tab, BatchGetParams& gp, const ReadLayout& lay,
                                  bool hash_outputs, const WholeFiles* wf = nullptr) {
  mec_codec* c = b->codec;
  const int k = gp.k, r = gp.r;
  const int64_t S = gp.S, P = gp.P, pitch = gp.pitch, nslots = lay.nslots();
  const int64_t stride = round_up(nslots * P + 512, 256);
  const bool raw = wf && wf->raw;
  if (!wf) mark_phase(b, s, 0);  // a batch with whole-file readers marks the start of its staging (batch_whole_stage)
  MEC_CUDA_OK(cudaMemcpyAsync(s.dreq.d.p, tab, lay.table_bytes, cudaMemcpyHostToDevice, s.st));
  int rc;
  if ((rc = s.aux.ensure(static_cast<size_t>(k * stride)))) return rc;
  if ((rc = s.out.ensure(static_cast<size_t>(nslots * std::max(r, 1) * pitch)))) return rc;
  if (!raw) {
    if ((rc = s.dig.d.ensure(static_cast<size_t>(nslots * (k + r) * 32)))) return rc;
    if ((rc = s.flags.ensure(static_cast<size_t>(nslots * k)))) return rc;
  }
  gp.arena = static_cast<uint8_t*>(s.aux.p); gp.arena_stride = stride;
  gp.rebuilt = static_cast<const uint8_t*>(s.out.p);
  const unsigned gx = static_cast<unsigned>(std::min<int64_t>(std::max<int64_t>(lay.max_nb, 1), 16));
  // long ranges are staged by the copy engines (k strided copies per request are cheap next to megabytes of frames); short ones by
  // the gather kernel (no per-request driver call at all)
  const int64_t fstride = 32 + S;
  if (wf) {
    batch_whole_rows_kernel<<<dim3(gx, static_cast<unsigned>(k), static_cast<unsigned>(gp.nreq)), 128, 0, s.st>>>(gp, wf->files, wf->streams,
                                                                                                                  wf->first);
    MEC_CUDA_OK(cudaGetLastError());
    c->eng->count_launch();
  }
  if (!raw) {
    // one 1-D copy per (request, survivor, block) frame — the arena pads frames to a 16-byte pitch — all of them in ONE batched call
    std::vector<void*> dsts, srcs;
    std::vector<size_t> sizes;
    bool any_gather = false;
    for (int q = 0; q < gp.nreq; q++) {
      const BatchGetDesc& d = tab[q];
      const uint32_t frames = ~d.whole_pos & ((1ull << k) - 1);  // positions with frames to stage
      if (!d.dma) { any_gather |= frames != 0; continue; }
      const int64_t nf = d.nblocks - (d.tail_slot >= 0 ? 1 : 0);
      for (int t = 0; t < k; t++) {
        if (!((frames >> t) & 1)) continue;
        const uint8_t* f = d.files[d.chosen[t]] + d.start_block * fstride;
        uint8_t* a = gp.arena + t * stride;
        for (int64_t j = 0; j < nf; j++) {
          dsts.push_back(a + (d.slot0 + j) * P); srcs.push_back(const_cast<uint8_t*>(f) + j * fstride); sizes.push_back(static_cast<size_t>(fstride));
        }
        if (d.tail_slot >= 0) {
          dsts.push_back(a + d.tail_slot * P); srcs.push_back(const_cast<uint8_t*>(f) + nf * fstride); sizes.push_back(static_cast<size_t>(32 + d.last_len));
        }
      }
    }
    if ((rc = copy_batch(dsts, srcs, sizes, s.st))) return rc;
    if (any_gather) {
      batch_get_gather_kernel<<<dim3(gx, static_cast<unsigned>(k), static_cast<unsigned>(gp.nreq)), 128, 0, s.st>>>(gp);
      MEC_CUDA_OK(cudaGetLastError());
      c->eng->count_launch();
    }
  }
  mark_phase(b, s, 1);
  if (!raw) MEC_CUDA_OK(cudaMemsetAsync(s.flags.d.p, 0, static_cast<size_t>(nslots * k), s.st));
  const int32_t* block_len = nullptr;
  const bool mixed = lay.npat > 1;
  const uint8_t* dtab = static_cast<const uint8_t*>(s.dreq.d.p);
  auto launch = [&](int64_t slot0, int64_t cnt, int64_t shard_len) -> int {
    FusedDesc d;
    d.block_len = block_len;
    if (mixed) {
      d.patterns = reinterpret_cast<const SmallPattern*>(dtab + lay.pat_off);
      d.block_pattern = reinterpret_cast<const uint16_t*>(dtab + lay.bp_off);
    }
    d.k = k; d.r = r; d.coef = lay.rows; d.static_encode = false; d.contiguous = false; d.hash_outputs = hash_outputs;
    d.key = kMagicKey; d.out_pitch = pitch; d.expect_block_stride = P; d.in_block_stride = P;
    d.nblocks = cnt; d.S = static_cast<int32_t>(shard_len);
    for (int t = 0; t < k; t++) {
      const uint8_t* base = gp.arena + t * stride + slot0 * P;
      d.map_base[t] = base; d.map_len[t] = stride - slot0 * P; d.expect_ptr[t] = base; d.in_ptr[t] = base + 32;
    }
    d.out = static_cast<uint8_t*>(s.out.p) + slot0 * r * pitch;
    if (!raw) {
      d.digests = static_cast<uint8_t*>(s.dig.d.p) + slot0 * (k + r) * 32;
      d.corrupt = static_cast<uint8_t*>(s.flags.d.p) + slot0 * k;
    }
    return c->eng->launch_fused(d, c->opt, s.st);
  };
  if (mixed && !c->eng->small_ok(c->opt, nslots)) return MEC_ERR_UNSUPPORTED;
  if (raw && r == 0) {
    // nothing to rebuild and nothing to verify: every request reads its k data drives
  } else if (mixed && lay.ntails == 0) {
    if ((rc = launch(0, nslots, S))) return rc;
  } else if (lay.ntails > 0 && c->eng->small_ok(c->opt, nslots)) {
    // ONE launch for every block of every caller, the short last ones included (per-block shard lengths in the latency kernel)
    if ((rc = s.blk.ensure(static_cast<size_t>(nslots) * sizeof(int32_t)))) return rc;
    int32_t* lens = static_cast<int32_t*>(s.blk.h.p);
    for (int64_t q = 0; q < lay.nfull_slots; q++) lens[q] = static_cast<int32_t>(S);
    for (int q = 0; q < gp.nreq; q++)
      if (tab[q].tail_slot >= 0) lens[tab[q].tail_slot] = static_cast<int32_t>(tab[q].last_len);
    MEC_CUDA_OK(s.blk.upload(static_cast<size_t>(nslots) * sizeof(int32_t), s.st));
    block_len = static_cast<const int32_t*>(s.blk.d.p);
    if ((rc = launch(0, nslots, S))) return rc;
  } else {
    if (lay.nfull_slots > 0 && (rc = launch(0, lay.nfull_slots, S))) return rc;  // ONE launch for every caller's full blocks
    for (int q = 0; q < gp.nreq; q++)
      if (tab[q].tail_slot >= 0 && (rc = launch(tab[q].tail_slot, 1, tab[q].last_len))) return rc;
  }
  if (!raw) MEC_CUDA_OK(s.flags.download(static_cast<size_t>(nslots * k), s.st));
  mark_phase(b, s, 2);
  b->st_patterns += lay.npat;
  if (mixed) b->st_mixed++;
  int64_t rebuilt = 0;
  for (int q = 0; q < gp.nreq; q++) rebuilt += tab[q].nblocks * tab[q].r;
  c->st_blocks_read += nslots;
  c->st_shards_rebuilt += rebuilt;
  return MEC_OK;
}

// one merged launch for the GETs of a batch that share a reader set (alive mask): gather kernel -> fused reconstruct over all full
// blocks (+ one launch per short last block) -> scatter kernel into every caller's destination
static int batcher_submit_get(mec_batcher* b, Slot& s, std::vector<BatchReq*>& reqs, int64_t* nblocks) {
  mec_codec* c = b->codec;
  BatchGetParams gp;
  ReadLayout lay;
  int rc = batch_read_plan(b, s, reqs, gp, lay);
  if (rc) return rc;
  const int k = gp.k, r = gp.r;
  const int64_t S = gp.S, P = gp.P, pitch = gp.pitch, nslots = lay.nslots();
  BatchGetDesc* tab = static_cast<BatchGetDesc*>(s.dreq.h.p);
  // writeDataBlocks: 0 = the scatter kernel assembles every object in device memory and ONE copy per request takes it to the caller
  // (fewest driver-side copy descriptors), 1 = the scatter kernel stores straight into the callers' buffers over PCIe, 2 = the copy
  // engine moves every (request, shard, block) piece itself
  // A batch with whole-file readers stages their shard files in s.src (batch_whole_stage), so it scatters straight into the callers'
  // buffers instead of assembling there.
  const bool whole = reqs.front()->whole_algo != 0;
  const int out_mode = whole && b->sw.get_out == 0 ? 1 : b->sw.get_out;
  // An encrypted GET's ciphertext range is assembled there in every mode, for sse_get_open (such a batch has no whole-file reader).
  std::vector<int64_t> asm_off(reqs.size(), -1);
  bool sse = false;
  for (const BatchReq* r : reqs) sse |= r->sse_key != nullptr;
  if (out_mode == 0 || sse) {
    int64_t total = 0;
    for (size_t q = 0; q < reqs.size(); q++)
      if (out_mode == 0 || reqs[q]->sse_key) { asm_off[q] = total; total += round_up(tab[q].length, 256); }
    if ((rc = s.src.ensure(static_cast<size_t>(total + 256)))) return rc;
    for (size_t q = 0; q < reqs.size(); q++)
      if (asm_off[q] >= 0) tab[q].dst = static_cast<uint8_t*>(s.src.p) + asm_off[q];
  }
  WholeFiles wf;
  if (whole && (rc = batch_whole_stage(b, s, reqs, tab, &wf))) return rc;
  if ((rc = batch_read_reconstruct(b, s, tab, gp, lay, false, whole ? &wf : nullptr))) return rc;  // GetObject reads no digest of rebuilt data
  const unsigned gx = static_cast<unsigned>(std::min<int64_t>(std::max<int64_t>(lay.max_nb, 1), 16));
  const int64_t stride = gp.arena_stride;
  if (out_mode == 2) {
    // writeDataBlocks by the copy engine: one 1-D copy per (request, data shard, block) piece, all in one batched call
    std::vector<void*> dsts, srcs;
    std::vector<size_t> sizes;
    int tpos[kMaxShards], qpos[kMaxShards];
    for (size_t rq = 0; rq < reqs.size(); rq++) {
      const BatchGetDesc& d = tab[rq];
      for (int i = 0; i < k; i++) { tpos[i] = qpos[i] = -1; }
      for (int t = 0; t < k; t++) if (d.chosen[t] < k) tpos[d.chosen[t]] = t;
      for (int q = 0; q < d.r; q++) qpos[d.targets[q]] = q;
      for (int64_t bb = 0; bb < d.nblocks; bb++) {
        const bool is_tail = d.tail_slot >= 0 && bb == d.nblocks - 1;
        const int64_t cur = is_tail ? d.last_len : S, slot = is_tail ? d.tail_slot : d.slot0 + bb;
        for (int i = 0; i < k; i++) {
          const DataSlice sl = data_slice(d.start_block + bb, i, cur, gp.bs, d.total, d.offset, d.offset + d.length);
          if (sl.e <= sl.a) continue;
          const uint8_t* src = tpos[i] >= 0 ? gp.arena + tpos[i] * stride + slot * P + 32 : gp.rebuilt + (slot * r + qpos[i]) * pitch;
          dsts.push_back(d.dst + (sl.a - d.offset)); srcs.push_back(const_cast<uint8_t*>(src) + sl.off); sizes.push_back(static_cast<size_t>(sl.e - sl.a));
        }
      }
    }
    if ((rc = copy_batch(dsts, srcs, sizes, s.st))) return rc;
  } else {
    batch_get_scatter_kernel<<<dim3(gx, static_cast<unsigned>(k), static_cast<unsigned>(reqs.size())), 128, 0, s.st>>>(gp);
    MEC_CUDA_OK(cudaGetLastError());
    c->eng->count_launch();
    if (out_mode == 0) {
      std::vector<void*> dsts, srcs;
      std::vector<size_t> sizes;
      for (size_t q = 0; q < reqs.size(); q++) {
        if (tab[q].length <= 0 || reqs[q]->sse_key) continue;
        dsts.push_back(reqs[q]->dst); srcs.push_back(static_cast<uint8_t*>(s.src.p) + asm_off[q]); sizes.push_back(static_cast<size_t>(tab[q].length));
      }
      if ((rc = copy_batch(dsts, srcs, sizes, s.st))) return rc;
    }
  }
  if (sse && (rc = sse_get_open(b, s, reqs, asm_off))) return rc;
  mark_phase(b, s, 3);
  *nblocks = nslots;
  return MEC_OK;
}

// one merged launch for the heals of a batch that share a reader set and a stale set: survivor frames staged as for GETs -> fused
// reconstruct of every stale shard, data and parity, with its digest (ONE latency launch when the batch is small enough, otherwise
// one over all full blocks plus one per short last block) -> the heal scatter kernel writes the healed frames into every caller's
// part-file images
static int batcher_submit_heal(mec_batcher* b, Slot& s, std::vector<BatchReq*>& reqs, int64_t* nblocks) {
  mec_codec* c = b->codec;
  BatchGetParams gp;
  ReadLayout lay;
  int rc = batch_read_plan(b, s, reqs, gp, lay);
  if (rc) return rc;
  const int r = gp.r;
  const int64_t nslots = lay.nslots();
  const BatchGetDesc* tab = static_cast<const BatchGetDesc*>(s.dreq.h.p);
  const bool whole = reqs.front()->whole_algo != 0;
  WholeFiles wf;
  if (whole) {
    if ((rc = batch_whole_stage(b, s, reqs, tab, &wf))) return rc;
    wf.raw = false;  // the healed frames carry the digests of the rebuilt shards
  }
  if ((rc = batch_read_reconstruct(b, s, tab, gp, lay, true, whole ? &wf : nullptr))) return rc;
  if (r > 0) {
    const unsigned gx = static_cast<unsigned>(std::min<int64_t>(std::max<int64_t>(lay.max_nb, 1), 16));
    batch_heal_scatter_kernel<<<dim3(gx, static_cast<unsigned>(r), static_cast<unsigned>(reqs.size())), 128, 0, s.st>>>(
        gp, static_cast<const uint8_t*>(s.dig.d.p), reinterpret_cast<uint8_t* const*>(gp.reqs + gp.nreq));
    MEC_CUDA_OK(cudaGetLastError());
    c->eng->count_launch();
  }
  mark_phase(b, s, 3);
  *nblocks = nslots;
  return MEC_OK;
}

// Device memory of a slot's batches with whole-file readers, for a batch of `slots` blocks and at most as many requests: request z
// of NB_z blocks stages at most k files of at most NB_z x S bytes (k x S < block_size + k), each padded by at most 15 + 256 bytes, so
// the file arena fits slots x (block_size + 272 x k) bytes; one stream-table entry, one first-stream index and one digest per file.
// A transcode batcher sizes this up front (batcher_create); any other batcher on a slot's first batch with whole-file readers.
static int size_whole_slot(const mec_codec* c, Slot& s, int64_t slots) {
  const int k = c->k;
  const size_t tab = static_cast<size_t>(slots * k) * sizeof(WholeStream) + static_cast<size_t>(slots) * sizeof(int32_t);
  int rc;
  if ((rc = s.src.ensure(static_cast<size_t>(slots * (c->block_size + 272 * k))))) return rc;
  if ((rc = s.wtab.ensure(tab))) return rc;
  return s.wdig.ensure(static_cast<size_t>(slots * k * 64));
}
// the blocks a batcher's slots are sized for (batcher_create)
static int64_t batcher_slot_blocks(const mec_batcher* b) { return b->max_blocks + std::min<int64_t>(64, b->max_blocks / 8 + 4); }

// The staging of the whole-file readers of a merged batch (every reader of a whole-file move, mec_batcher_transcode_whole; the
// whole-file readers among a mixed GET's or heal's k chosen, mec_batcher_decode_mixed / _heal_mixed), on the slot's stream: the raw
// shard files of every request's whole-file positions (bit t of tab[z].whole_pos: reader tab[z].chosen[t]) -> the file arena in
// s.src (each 16-byte aligned with 256 readable bytes behind it, as stage_verified_whole lays files out) in ONE batched copy, then
// ONE whole_hash_kernel launch over a stream table that holds only those files, in request order and ascending position order
// within a request, and their digests back to s.wdig.h, where batcher_finish compares them with every request's expected sums.
// Request z's first stream is first[z], stored behind the stream table.  s.src is free: a heal or move batch does not stage object
// bytes, and a GET batch with whole-file readers scatters straight into its callers' buffers (batcher_submit_get).  Counts
// "bytes_h2d" as mec_decode_mixed does: the frames of every streaming reader plus one shard file per whole-file reader.
static int batch_whole_stage(mec_batcher* b, Slot& s, const std::vector<BatchReq*>& reqs, const BatchGetDesc* tab, WholeFiles* wf) {
  mec_codec* c = b->codec;
  const int k = c->k;
  const size_t nreq = reqs.size();
  int rc;
  if ((rc = size_whole_slot(c, s, batcher_slot_blocks(b)))) return rc;  // a no-op after the slot's first such batch
  size_t nfiles = 0;
  for (size_t z = 0; z < nreq; z++) nfiles += static_cast<size_t>(__builtin_popcount(tab[z].whole_pos));
  const size_t tab_bytes = nfiles * sizeof(WholeStream) + nreq * sizeof(int32_t);
  if ((rc = s.wtab.ensure(tab_bytes))) return rc;  // a request larger than the slots' sizing leads its own batch
  if ((rc = s.wdig.ensure(nfiles * 64))) return rc;
  WholeStream* ws = static_cast<WholeStream*>(s.wtab.h.p);
  int32_t* first = reinterpret_cast<int32_t*>(ws + nfiles);
  int64_t arena = 0;
  size_t j = 0;
  for (size_t z = 0; z < nreq; z++) {
    const BatchGetDesc& d = tab[z];
    const int64_t sfs = mec_shard_file_size(c, d.total);
    const int nw = __builtin_popcount(d.whole_pos);
    first[z] = static_cast<int32_t>(j);
    for (int t = 0; t < k; t++)
      if ((d.whole_pos >> t) & 1) {
        ws[j++] = WholeStream{arena, sfs};
        arena += round_up(sfs, 16) + 256;
      }
    const FrameGeom g{d.nblocks, c->S(), d.last_len};
    c->st_h2d += nw * sfs + (k - nw) * g.file_bytes();
  }
  if ((rc = s.src.ensure(static_cast<size_t>(arena)))) return rc;
  uint8_t* files = static_cast<uint8_t*>(s.src.p);
  mark_phase(b, s, 0);
  MEC_CUDA_OK(s.wtab.upload(tab_bytes, s.st));
  std::vector<void*> dsts, srcs;
  std::vector<size_t> sizes;
  j = 0;
  for (size_t z = 0; z < nreq; z++)
    for (int t = 0; t < k; t++)
      if ((tab[z].whole_pos >> t) & 1) {
        const WholeStream& w = ws[j++];
        if (w.len == 0) continue;
        dsts.push_back(files + w.off); srcs.push_back(const_cast<uint8_t*>(tab[z].files[tab[z].chosen[t]])); sizes.push_back(static_cast<size_t>(w.len));
      }
  if ((rc = copy_batch(dsts, srcs, sizes, s.st))) return rc;
  const WholeStream* dws = static_cast<const WholeStream*>(s.wtab.d.p);
  if ((rc = whole_hash_device(c, reqs.front()->whole_algo, files, 0, 0, static_cast<int64_t>(nfiles), static_cast<uint8_t*>(s.wdig.d.p), s.st, dws)))
    return rc;
  c->eng->count_launch();
  MEC_CUDA_OK(s.wdig.download(nfiles * 64, s.st));
  bool streaming = false;  // a request of the batch reads frames
  for (size_t z = 0; z < nreq; z++) streaming |= tab[z].whole_pos != static_cast<uint32_t>((1ull << k) - 1);
  *wf = WholeFiles{files, dws, reinterpret_cast<const int32_t*>(dws + nfiles), !streaming};
  return MEC_OK;
}

// one merged batch of moves between pools (mec_batcher_transcode), everything on the source slot's stream: survivor frames staged and
// the missing data shards rebuilt as for whole-part GETs (not hashed: they are consumed here) -> batch_transcode_resplit_kernel
// writes every request's object bytes into the destination slot's staging in the PUT layout -> the destination codec's encode and
// frame scatter of a merged PUT batch into every caller's out files.  The destination codec's slot with the same index holds the
// destination side (as emit_transcode uses it), so the six batches in flight never share staging.  A batch of whole-file moves
// (mec_batcher_transcode_whole) is staged and hashed by batch_whole_stage and its raw shard rows laid into the frame arena; from the
// rebuild on it runs exactly as a batch of streaming moves.
static int batcher_submit_transcode(mec_batcher* b, Slot& s, std::vector<BatchReq*>& reqs, int64_t* nblocks) {
  mec_codec* c = b->codec;
  mec_codec* e = b->dst;
  Slot& d = e->slots[&s - c->slots];
  const bool whole = reqs.front()->kind == ReqKind::TranscodeWhole;
  BatchGetParams gp;
  ReadLayout lay;
  int rc = batch_read_plan(b, s, reqs, gp, lay);
  if (rc) return rc;
  PutLayout put;  // every request's destination side: a PUT of the part (mec_batcher_transcode)
  if ((rc = put_layout(e, d, reqs, true, false, put))) return rc;
  const size_t nreq = reqs.size();
  const int ek = e->k, en = e->n;
  const int64_t bs = e->block_size, eS = e->S(), epitch = round_up(eS, 16);
  for (const BatchReq* r : reqs) {
    const int64_t nf = r->total / bs, tl = r->total % bs;
    if (!whole)
      c->st_h2d += static_cast<int64_t>(c->k) * mec_bitrot_shard_file_size(mec_shard_file_size(c, r->total), c->S(), MEC_HIGHWAYHASH256S);
    e->st_d2h += (nf * eS + (tl ? ceil_frac(tl, ek) : 0)) * en;
  }
  const BatchReqDesc* dt = static_cast<const BatchReqDesc*>(d.dreq.h.p);
  const BatchGetDesc* rt = static_cast<const BatchGetDesc*>(s.dreq.h.p);
  WholeFiles wf;
  if (whole && (rc = batch_whole_stage(b, s, reqs, rt, &wf))) return rc;  // every reader whole-file: wf.raw
  if ((rc = batch_read_reconstruct(b, s, rt, gp, lay, false, whole ? &wf : nullptr))) return rc;
  MEC_CUDA_OK(d.dreq.upload(nreq * sizeof(BatchReqDesc), s.st));
  BatchCopyParams cp;
  cp.reqs = static_cast<const BatchReqDesc*>(d.dreq.d.p);
  cp.nreq = static_cast<int>(nreq); cp.k = ek; cp.m = e->m; cp.bs = bs; cp.S = eS; cp.pitch = epitch;
  cp.staged = static_cast<uint8_t*>(d.src.p); cp.parity = static_cast<const uint8_t*>(d.out.p); cp.digests = static_cast<const uint8_t*>(d.dig.d.p);
  const unsigned gx = static_cast<unsigned>(std::min<int64_t>(std::max<int64_t>(lay.max_nb, 1), 16));
  batch_transcode_resplit_kernel<<<dim3(gx, static_cast<unsigned>(c->k), static_cast<unsigned>(nreq)), 128, 0, s.st>>>(gp, cp);
  MEC_CUDA_OK(cudaGetLastError());
  c->eng->count_launch();
  if ((rc = batch_encode_scatter(e, d, s.st, dt, nreq, put, cp, nullptr))) return rc;
  mark_phase(b, s, 3);
  e->st_blocks_encoded += put.nslots;
  *nblocks = lay.nslots();
  return MEC_OK;
}

// What one merged verify batch may hold: frames for one hash-only launch (the latency kernel's limit; with options that rule it out,
// the blocks a slot is sized for), staged bytes within the slot's PUT staging buffer, whole-file parts within the stream table
// size_whole_slot sizes.  A call beyond any of them takes the private path.
struct VerifyLimits {
  int64_t frames, bytes, files;
};
static VerifyLimits verify_limits(const mec_batcher* b) {
  const mec_codec* c = b->codec;
  const int64_t slots = batcher_slot_blocks(b);
  return VerifyLimits{c->eng->small_ok(c->opt, 1) ? c->eng->small_limit(c->opt) : slots, slots * c->block_size - 1024, slots * c->k};
}

// One merged batch of verify calls (mec_batcher_verify), on the slot's stream: every frame of every streaming part (frame j at
// s.src + j * P) and every whole-file part (from round_up(nframes * P + 512, 256) on, each 16-byte aligned with 256 readable bytes
// behind it, as batch_whole_stage lays files out) in ONE batched copy; ONE hash-only launch over every frame with the per-frame
// length table (verify_frames); ONE whole_hash_kernel launch whose algorithm groups hold every whole-file part (verify_whole_firsts'
// order); the frame verdicts and file digests back to s.flags.h and s.wdig.h, where batcher_finish folds them into each caller's
// results.  Nothing is redone: a corrupt part is a result.
static int batcher_submit_verify(mec_batcher* b, Slot& s, const std::vector<BatchReq*>& reqs, int64_t* nblocks) {
  mec_codec* c = b->codec;
  const int64_t S = c->S(), fstride = 32 + S, P = round_up(32 + S, 16);
  int64_t nframes = 0, nwhole = 0, next[kWholeGroups], counts[kWholeGroups];
  for (const BatchReq* r : reqs) { nframes += r->vframes; nwhole += r->vwhole; }
  verify_whole_firsts(reqs, next);
  for (int g = 0; g < kWholeGroups; g++) counts[g] = (g + 1 < kWholeGroups ? next[g + 1] : nwhole) - next[g];
  int rc;
  if (nwhole > 0 && (rc = size_whole_slot(c, s, batcher_slot_blocks(b)))) return rc;  // a no-op after the slot's first such batch
  const int64_t woff = round_up(nframes * P + 512, 256);
  int64_t end = woff;
  for (const BatchReq* r : reqs) end += r->vbytes - r->vframes * P;  // the whole-file parts (verify_staged)
  if ((rc = s.src.ensure(static_cast<size_t>(end)))) return rc;
  if ((rc = s.dreq.h.ensure(static_cast<size_t>(nframes) * sizeof(int32_t) + 16))) return rc;
  if ((rc = s.wtab.ensure(static_cast<size_t>(nwhole) * sizeof(WholeStream) + 16)))
    return rc;
  if ((rc = s.wdig.ensure(static_cast<size_t>(nwhole) * 64 + 64))) return rc;
  uint8_t* arena = static_cast<uint8_t*>(s.src.p);
  int32_t* lens = static_cast<int32_t*>(s.dreq.h.p);
  WholeStream* ws = static_cast<WholeStream*>(s.wtab.h.p);
  CopyList list;
  int64_t f = 0, wpos = woff;
  for (const BatchReq* r : reqs)
    for (int64_t p = 0; p < r->vparts; p++) {
      if (r->vresults[p] != MEC_OK) continue;
      const int a = r->valgos[p];
      const uint8_t* file = r->vfiles[p];
      if (a == MEC_HIGHWAYHASH256S) {
        const int64_t nb = ceil_frac(r->vpart_lens[p], S), last = r->vpart_lens[p] - (nb - 1) * S;
        for (int64_t j = 0; j < nb; j++, f++) {
          lens[f] = static_cast<int32_t>(j == nb - 1 ? last : S);
          list.add(arena + f * P, file + j * fstride, 32 + lens[f]);
        }
        c->st_h2d += r->vfile_lens[p];
      } else {
        const int64_t len = r->vfile_lens[p];
        ws[next[whole_group(a)]++] = WholeStream{wpos, len};
        list.add(arena + wpos, file, len);
        wpos += round_up(len, 16) + 256;
        c->st_h2d += len;
      }
    }
  mark_phase(b, s, 0);
  if (nwhole > 0)
    MEC_CUDA_OK(s.wtab.upload(static_cast<size_t>(nwhole) * sizeof(WholeStream), s.st));
  if ((rc = list.flush(s.st))) return rc;
  mark_phase(b, s, 1);
  if (nframes > 0 && (rc = verify_frames(c, s, arena, nframes, nframes, lens, c->eng->small_ok(c->opt, nframes)))) return rc;
  if (nwhole > 0) {
    if ((rc = whole_hash_groups(c, kWholeGroups, kWholeAlgos, counts, arena, 0, 0, static_cast<uint8_t*>(s.wdig.d.p), s.st,
                                static_cast<const WholeStream*>(s.wtab.d.p))))
      return rc;
    c->eng->count_launch();
    MEC_CUDA_OK(s.wdig.download(static_cast<size_t>(nwhole) * 64, s.st));
  }
  mark_phase(b, s, 2);
  mark_phase(b, s, 3);
  *nblocks = nframes;
  return MEC_OK;
}

static void batcher_main(mec_batcher* b) {
  mec_codec* c = b->codec;
  cudaSetDevice(c->device);
  InflightBatch inflight[kSlots];
  int head = 0, tail = 0, nbusy = 0;
  using clk = std::chrono::steady_clock;
  auto us_since = [](clk::time_point t0) { return std::chrono::duration_cast<std::chrono::microseconds>(clk::now() - t0).count(); };
  for (;;) {
    std::vector<BatchReq*> reqs;
    {
      std::unique_lock<std::mutex> lk(b->mu);
      const auto t_idle = clk::now();
      if (nbusy == 0) b->cv_work.wait(lk, [&] { return b->stop || !b->queue.empty(); });
      b->us_idle += us_since(t_idle);
      if (b->stop && b->queue.empty() && nbusy == 0) return;
      if (!b->queue.empty() && nbusy < kSlots) {
        // gather: whatever is queued now; when nothing is in flight, give concurrent callers max_wait_us to join
        auto req_blocks = [&](const BatchReq* r) -> int64_t {
          // heal, transcode, a GET with a whole-file reader (its shard files are staged whole): the whole part
          // a verify: its staged bytes
          return r->kind == ReqKind::Put                      ? ceil_frac(r->len, c->block_size)
                 : r->kind == ReqKind::Verify                 ? ceil_frac(r->vbytes, c->block_size)
                 : r->kind == ReqKind::Get && !r->whole_algo ? r->length / c->block_size + 2
                                                              : ceil_frac(r->total, c->block_size);
        };
        auto blocks_queued = [&] {
          int64_t nb = 0;
          for (BatchReq* r : b->queue) nb += req_blocks(r);
          return nb;
        };
        // an idle GPU gives the first caller up to max_wait_us of company before its batch is cut
        // (waiting while batches are in flight only adds latency to a closed loop of callers)
        if (nbusy == 0 && b->max_wait_us > 0 && blocks_queued() < b->max_blocks)
          b->cv_work.wait_for(lk, std::chrono::microseconds(b->max_wait_us), [&] { return b->stop || blocks_queued() >= b->max_blocks; });
        // a batch = the oldest request plus everything queued behind it of the same kind (and, for GETs, heals and transcodes, the same reader
        // set; for heals also the same stale drives — unless b->mix: then reads of other patterns join while the batch's blocks fit
        // one latency launch, and a batch of several patterns is cut at that limit; whole-file moves also share their algorithm)
        // a shallow pipeline is filled with several smaller batches rather than one big one: the fused kernel takes ~0.45 ms however few
        // blocks it is given (one warp walks one erasure block), so the copy of one batch has to overlap the kernel of another —
        // otherwise a closed loop of callers falls into a convoy (all of them in one batch, the GPU idle while they wake up)
        const int depth = b->sw.depth;
        int64_t cap = b->max_blocks;
        if (depth > 0 && nbusy < depth - 1) {
          const int64_t q = blocks_queued();
          if (q > 8) cap = std::min(cap, std::max<int64_t>(4, ceil_frac(q, depth - nbusy)));
        }
        int64_t nb = 0, nread = 0;
        bool mixed = false;
        const BatchReq* lead = b->queue.front();
        const bool mix = b->mix && is_read(lead->kind);
        const int64_t limit = std::min<int64_t>(c->eng->small_limit(c->opt), 1 << 16);  // block_pattern holds uint16_t indices
        // verify batches: calls with a whole-file part only with such calls (a frame-only scan never waits behind the chain hash of a
        // long legacy file), cut at verify_limits
        const VerifyLimits vlim = verify_limits(b);
        int64_t vframes = 0, vbytes = 0, vwhole = 0;
        for (auto it = b->queue.begin(); it != b->queue.end();) {
          BatchReq* r = *it;
          const bool same = r->alive_mask == lead->alive_mask && r->stale_mask == lead->stale_mask;
          if (r->kind != lead->kind || r->whole_algo != lead->whole_algo || (!same && !mix) || (r->vwhole > 0) != (lead->vwhole > 0)) {
            ++it;
            continue;
          }
          const int64_t rb = req_blocks(r);
          if (!reqs.empty() && nb + rb > cap) break;
          if (r->kind == ReqKind::Verify) {
            if (!reqs.empty() && (vframes + r->vframes > vlim.frames || vbytes + r->vbytes > vlim.bytes || vwhole + r->vwhole > vlim.files)) break;
            vframes += r->vframes; vbytes += r->vbytes; vwhole += r->vwhole;
          }
          if (mix) {  // the exact blocks of the read
            const int64_t rs = read_range(c, r->offset, r->length, r->total).nblocks;
            if ((mixed || !same) && nread + rs > limit) break;
            mixed |= !same;
            nread += rs;
          }
          reqs.push_back(r);
          it = b->queue.erase(it);
          nb += rb;
        }
      }
    }
    if (!reqs.empty()) {
      Slot& s = c->slots[head];
      InflightBatch& fb = inflight[head];
      int rc = MEC_OK;
      int64_t nblocks = 0;
      const auto t_submit = clk::now();
      fb.kind = reqs.front()->kind;
      {
        std::lock_guard<std::mutex> lk(c->mu);
        switch (fb.kind) {
          case ReqKind::Put: rc = batcher_submit(b, s, reqs, &fb.needs_retire, &nblocks); break;
          case ReqKind::Get: rc = batcher_submit_get(b, s, reqs, &nblocks); break;
          case ReqKind::Heal: rc = batcher_submit_heal(b, s, reqs, &nblocks); break;
          case ReqKind::Verify: rc = batcher_submit_verify(b, s, reqs, &nblocks); break;
          case ReqKind::Transcode:
          case ReqKind::TranscodeWhole: {
            std::lock_guard<std::mutex> lk_dst(b->dst->mu);  // source, then destination: mec_transcode's order
            rc = batcher_submit_transcode(b, s, reqs, &nblocks);
            break;
          }
        }
      }
      b->us_submit += us_since(t_submit);
      fb.reqs = reqs;
      // a batch the kernels carry end to end: every read or verify batch, a PUT batch unless it took the memcpy path
      const bool kernel_batch = fb.kind != ReqKind::Put || !fb.needs_retire;
      fb.traced = b->sw.trace && rc == MEC_OK && kernel_batch;
      if (rc != MEC_OK) {  // drain what was enqueued before the failure, then fail the whole batch
        if (s.sse_keys.p) cudaMemsetAsync(s.sse_keys.p, 0, s.sse_keys.cap, s.st);  // a failure between key setup and cipher
        cudaStreamSynchronize(s.st);
        if (b->sum_st[head]) cudaStreamSynchronize(b->sum_st[head]);
        batcher_finish(b, fb, s, rc);
      } else {
        b->st_batches++;
        if (kernel_batch) b->st_kernel_batches++;
        b->st_requests += static_cast<int64_t>(reqs.size());
        b->st_blocks += nblocks;
        head = (head + 1) % kSlots;
        nbusy++;
      }
      bool more;
      {
        std::lock_guard<std::mutex> lk(b->mu);
        more = !b->queue.empty();
      }
      if (more && nbusy < kSlots) continue;  // keep the slots full before waiting on the oldest batch
    }
    if (nbusy > 0) {
      const auto t_sync = clk::now();
      const cudaError_t e = cudaStreamSynchronize(c->slots[tail].st);
      b->us_sync += us_since(t_sync);
      if (inflight[tail].traced && e == cudaSuccess) {
        float a = 0, k2 = 0, sc = 0;
        cudaEventElapsedTime(&a, b->ev_ph[tail][0], b->ev_ph[tail][1]);
        cudaEventElapsedTime(&k2, b->ev_ph[tail][1], b->ev_ph[tail][2]);
        cudaEventElapsedTime(&sc, b->ev_ph[tail][2], b->ev_ph[tail][3]);
        b->us_stage += static_cast<int64_t>(a * 1000); b->us_kernel += static_cast<int64_t>(k2 * 1000); b->us_scatter += static_cast<int64_t>(sc * 1000);
      }
      const auto t_fin = clk::now();
      batcher_finish(b, inflight[tail], c->slots[tail], e == cudaSuccess ? MEC_OK : MEC_ERR_CUDA);
      b->us_finish += us_since(t_fin);
      tail = (tail + 1) % kSlots;
      nbusy--;
    }
  }
}
}  // namespace

// The environment switches of a new batcher (BatcherSwitches)
static BatcherSwitches batcher_switches() {
  BatcherSwitches w;
  const char* e;
  w.memcpy = getenv("MEC_BATCHER_MEMCPY") != nullptr;
  w.gather = getenv("MEC_BATCHER_GATHER") != nullptr;
  if ((e = getenv("MEC_BATCHER_GATHER_PCT"))) w.gather_pct = std::max(0, std::min(100, atoi(e)));
  if ((e = getenv("MEC_BATCHER_DMA_BLOCKS"))) w.dma_blocks = atoll(e);
  if ((e = getenv("MEC_BATCHER_GET_OUT"))) w.get_out = atoi(e);
  if ((e = getenv("MEC_BATCHER_DEPTH"))) w.depth = atoi(e);
  w.trace = getenv("MEC_BATCHER_TRACE") != nullptr;
  return w;
}

// Slot `s` of codec `c` sized up front for a merged PUT batch of `blocks` blocks: object bytes, parity rows, digests
static int size_put_slot(const mec_codec* c, Slot& s, int64_t blocks) {
  int rc;
  if ((rc = s.src.ensure(static_cast<size_t>(blocks * c->block_size)))) return rc;
  if ((rc = s.out.ensure(static_cast<size_t>(blocks * std::max(c->m, 1) * round_up(c->S(), 16))))) return rc;
  return s.dig.d.ensure(static_cast<size_t>(blocks * c->n * 32));
}

// mec_batcher_new_ex, and with `dst` (a codec of the destination geometry without an engine yet, owned from here on, freed on
// failure) mec_batcher_new_transcode: the destination's engine and slots are set up before the worker starts
static int batcher_create(int k, int m, int64_t block_size, int device, int64_t max_batch_blocks, int max_wait_us, int flags,
                          mec_codec* dst, mec_batcher** out) {
  std::unique_ptr<mec_batcher> b(new mec_batcher);
  b->dst = dst;
  int rc = mec_codec_new(k, m, block_size, MEC_HIGHWAYHASH256S, device, &b->codec);
  if (rc) return rc;
  mec_codec* c = b->codec;
  {
    std::lock_guard<std::mutex> lk(c->mu);
    rc = ensure_engine(c);
  }
  if (rc == MEC_OK && dst) {
    std::lock_guard<std::mutex> lk(dst->mu);
    rc = ensure_engine(dst);
  }
  if (rc == MEC_OK && (c->S() >= (1ll << 31) || (dst && dst->S() >= (1ll << 31)))) rc = MEC_ERR_UNSUPPORTED;
  if (rc) return rc;
  b->sw = batcher_switches();
  b->mix = (flags & MEC_BATCHER_MIX_PATTERNS) && c->eng->small_ok(c->opt, 1);  // per-block decode plans exist in the latency kernel only
  if (max_batch_blocks > 0) b->max_blocks = max_batch_blocks;
  // a merged batch stages at most 1 GiB of object bytes: six slots are sized for a full batch up front (below)
  b->max_blocks = std::max<int64_t>(1, std::min<int64_t>(b->max_blocks, (1ll << 30) / std::max<int64_t>(block_size, 1)));
  if (max_wait_us >= 0) b->max_wait_us = max_wait_us;
  {
    // size every slot for a full batch up front: growing a buffer later means cudaFree + cudaMalloc, which stall the whole device
    // (all six batches in flight) for tens of milliseconds — seen as p99 spikes of hundreds of ms before
    std::lock_guard<std::mutex> lk(c->mu);
    int cur = 0;
    cudaGetDevice(&cur);
    cudaSetDevice(device);
    const int64_t P = round_up(32 + c->S(), 16), slots = batcher_slot_blocks(b.get());
    for (Slot& s : c->slots) {
      if (rc == MEC_OK) rc = size_put_slot(c, s, slots);
      if (rc == MEC_OK) rc = s.dig.h.ensure(static_cast<size_t>(slots * c->n * 32));
      if (rc == MEC_OK) rc = s.aux.ensure(static_cast<size_t>(k * round_up(slots * P + 512, 256)));
      if (rc == MEC_OK) rc = s.flags.ensure(static_cast<size_t>(slots * k));
      // request tables: PUT rows, or GET rows, or GET rows plus one out-file pointer per rebuilt shard (heal); reads of several
      // erasure patterns add a pattern (at most one per request) and a pattern index per block
      const size_t row = std::max(sizeof(BatchReqDesc), sizeof(BatchGetDesc) + kMaxR * sizeof(uint8_t*) +
                                                            (b->mix ? sizeof(SmallPattern) + sizeof(uint16_t) : 0));
      if (rc == MEC_OK) rc = s.dreq.ensure(static_cast<size_t>(slots) * row + 16);
      // object checksums (batcher_crc_enqueue): a batch of at most `slots` requests and slots x block_size bytes has at most
      // slots x block_size / kCrcRegion whole regions plus two partial ones (full-block segment, short block) per request
      const int64_t nwork = ceil_frac(slots * block_size, kCrcRegion) + 2 * slots;
      const size_t tab = static_cast<size_t>(slots) * sizeof(CrcReq) + static_cast<size_t>(nwork) * sizeof(CrcWork);
      if (rc == MEC_OK) rc = s.crc_tab.ensure(tab);
      if (rc == MEC_OK) rc = s.crc_part.ensure(static_cast<size_t>(nwork) * kCrcTypes * sizeof(uint64_t));
      if (rc == MEC_OK) rc = s.crc_out.ensure(static_cast<size_t>(slots) * kCrcTypes * sizeof(uint64_t));
      // object hashes (batcher_sums_table): at most `slots` requests, each with up to kSumAlgos items and one record
      if (rc == MEC_OK) rc = s.sum_tab.ensure(static_cast<size_t>(slots) * kSumAlgos * sizeof(SumWork));
      if (rc == MEC_OK) rc = s.sum_out.ensure(static_cast<size_t>(slots) * kSumRecord);
    }
    for (int i = 0; i < kSlots && rc == MEC_OK; i++)
      if (b->sum_st[i].create(cudaStreamNonBlocking) != cudaSuccess || b->ev_staged[i].create(cudaEventDisableTiming) != cudaSuccess ||
          b->ev_summed[i].create(cudaEventDisableTiming) != cudaSuccess) {
        set_last_error(std::string("object-hash stream: ") + cudaGetErrorString(cudaGetLastError()));
        rc = MEC_ERR_CUDA;
      }
    if (rc == MEC_OK) rc = ensure_crc(c);
    if (dst)
      // merged whole-file moves (batch_whole_stage): the raw shard files of a batch in s.src (size_whole_slot)
      for (Slot& s : c->slots)
        if (rc == MEC_OK) rc = size_whole_slot(c, s, slots);
    if (dst) {
      // the destination side of a merged transcode batch, laid out as a merged PUT batch of the destination geometry: object bytes,
      // parity rows, digests, the PUT request table and the latency kernel's block table.  A batch of `slots` source blocks holds
      // the object bytes of slots x R destination blocks (R = block_size / dst block size); it has at most `slots` requests.
      std::lock_guard<std::mutex> lk_dst(dst->mu);
      const int64_t dslots = slots * (block_size / dst->block_size);
      for (Slot& s : dst->slots) {
        if (rc == MEC_OK) rc = size_put_slot(dst, s, dslots);
        if (rc == MEC_OK) rc = s.dreq.ensure(static_cast<size_t>(slots) * sizeof(BatchReqDesc) + 16);
        if (rc == MEC_OK) rc = s.blk.ensure(static_cast<size_t>(dslots) * sizeof(SmallBlock));
      }
    }
    cudaSetDevice(cur);
  }
  if (rc) return rc;
  if (b->sw.trace) {
    int cur = 0;
    cudaGetDevice(&cur);
    cudaSetDevice(device);
    for (int i = 0; i < kSlots; i++)
      for (int j = 0; j < 4; j++)
        if (b->ev_ph[i][j].create(cudaEventDefault) != cudaSuccess) { cudaGetLastError(); b->sw.trace = false; }
    cudaSetDevice(cur);
  }
  if (b->sw.gather_pct > 0) {
    int cur = 0;
    cudaGetDevice(&cur);
    cudaSetDevice(device);
    bool ok = b->aux.create(cudaStreamNonBlocking) == cudaSuccess;
    for (int i = 0; ok && i < kSlots; i++)
      ok = b->ev_table[i].create(cudaEventDisableTiming) == cudaSuccess && b->ev_gather[i].create(cudaEventDisableTiming) == cudaSuccess;
    cudaSetDevice(cur);
    if (!ok) { cudaGetLastError(); b->sw.gather_pct = 0; }
  }
  b->worker = std::thread(batcher_main, b.get());
  *out = b.release();
  return MEC_OK;
}
extern "C" int mec_batcher_new_ex(int k, int m, int64_t block_size, int device, int64_t max_batch_blocks, int max_wait_us, int flags,
                                  mec_batcher** out) {
  if (!out) return MEC_ERR_INVALID_ARGUMENT;
  *out = nullptr;
  if (flags & ~MEC_BATCHER_MIX_PATTERNS) return MEC_ERR_INVALID_ARGUMENT;
  return batcher_create(k, m, block_size, device, max_batch_blocks, max_wait_us, flags, nullptr, out);
}
extern "C" int mec_batcher_new_transcode_ex(int k, int m, int64_t block_size, int dst_k, int dst_m, int64_t dst_block_size, int device,
                                            int64_t max_batch_blocks, int max_wait_us, int flags, mec_batcher** out) {
  if (!out) return MEC_ERR_INVALID_ARGUMENT;
  *out = nullptr;
  mec_codec* probe = nullptr;
  int rc = mec_codec_new(k, m, block_size, MEC_HIGHWAYHASH256S, device, &probe);  // the source geometry's errors come first
  mec_codec_free(probe);
  if (rc) return rc;
  if ((rc = mec_codec_new(dst_k, dst_m, dst_block_size, MEC_HIGHWAYHASH256S, device, &probe))) return rc;
  mec_codec* dst = probe;
  if (flags & ~MEC_BATCHER_MIX_PATTERNS) { mec_codec_free(dst); return MEC_ERR_INVALID_ARGUMENT; }
  if (block_size % dst_block_size != 0) { mec_codec_free(dst); return MEC_ERR_UNSUPPORTED; }  // as mec_transcode
  return batcher_create(k, m, block_size, device, max_batch_blocks, max_wait_us, flags, dst, out);
}
extern "C" int mec_batcher_new_transcode(int k, int m, int dst_k, int dst_m, int64_t block_size, int device, int64_t max_batch_blocks,
                                         int max_wait_us, int flags, mec_batcher** out) {
  if (!out) return MEC_ERR_INVALID_ARGUMENT;
  *out = nullptr;
  if (flags & ~MEC_BATCHER_MIX_PATTERNS) return MEC_ERR_INVALID_ARGUMENT;  // this call has always refused unknown flags first
  return mec_batcher_new_transcode_ex(k, m, block_size, dst_k, dst_m, block_size, device, max_batch_blocks, max_wait_us, flags, out);
}
extern "C" int mec_batcher_new(int k, int m, int64_t block_size, int device, int64_t max_batch_blocks, int max_wait_us, mec_batcher** out) {
  return mec_batcher_new_ex(k, m, block_size, device, max_batch_blocks, max_wait_us, 0, out);
}

extern "C" void mec_batcher_free(mec_batcher* b) {
  if (!b) return;
  {
    std::lock_guard<std::mutex> lk(b->mu);
    b->stop = true;
  }
  b->cv_work.notify_all();
  if (b->worker.joinable()) b->worker.join();
  delete b;
}

// Queues `r` for the worker and waits until its batch is done.  A PUT wakes the worker only as the first arrival or as the one that
// fills a batch, not as every caller; a GET, heal or transcode always wakes it.
static int64_t batcher_enqueue_wait(mec_batcher* b, BatchReq& r) {
  std::unique_lock<std::mutex> lk(b->mu);
  if (b->stop) return MEC_ERR_INVALID_ARGUMENT;
  b->queue.push_back(&r);
  if (r.kind != ReqKind::Put || b->queue.size() == 1 ||
      static_cast<int64_t>(b->queue.size()) * std::max<int64_t>(1, r.len / b->codec->block_size) >= b->max_blocks)
    b->cv_work.notify_one();
  r.cv.wait(lk, [&] { return r.done; });
  return r.result;
}

static int64_t batcher_call(mec_batcher* b, const uint8_t* src, int64_t len, uint8_t* const* files, uint8_t* data_digests, bool with_data,
                            int write_quorum, int crc_which = 0, uint64_t* crc_out = nullptr, int sum_which = 0, uint8_t* sums = nullptr) {
  if (!b || len < 0 || !files || (len > 0 && !src)) return MEC_ERR_INVALID_ARGUMENT;
  int online = 0;
  for (int i = 0; i < b->codec->n; i++) online += files[i] != nullptr;
  if (online < write_quorum) return MEC_ERR_WRITE_QUORUM;  // cmd/erasure-encode.go:59-65
  if (len == 0) {  // cmd/erasure-coding.go:78-80; the checksums of the empty stream
    if (crc_which) {
      for (int ty = 0; ty < kCrcTypes; ty++) crc_out[ty] = 0;
      b->st_crc_requests++;
    }
    if (sum_which) {  // the digests of the empty message
      static const uint8_t kEmpty[kSumAlgos][32] = {
          {0xd4, 0x1d, 0x8c, 0xd9, 0x8f, 0x00, 0xb2, 0x04, 0xe9, 0x80, 0x09, 0x98, 0xec, 0xf8, 0x42, 0x7e},
          {0xda, 0x39, 0xa3, 0xee, 0x5e, 0x6b, 0x4b, 0x0d, 0x32, 0x55, 0xbf, 0xef, 0x95, 0x60, 0x18, 0x90, 0xaf, 0xd8, 0x07, 0x09},
          {0xe3, 0xb0, 0xc4, 0x42, 0x98, 0xfc, 0x1c, 0x14, 0x9a, 0xfb, 0xf4, 0xc8, 0x99, 0x6f, 0xb9, 0x24,
           0x27, 0xae, 0x41, 0xe4, 0x64, 0x9b, 0x93, 0x4c, 0xa4, 0x95, 0x99, 0x1b, 0x78, 0x52, 0xb8, 0x55}};
      for (int a = 0; a < kSumAlgos; a++)
        if (sum_which & (MEC_SUM_MD5 << a)) memcpy(sums + 32 * a, kEmpty[a], static_cast<size_t>(sum_digest_len(a)));
      b->st_sum_requests++;
    }
    return 0;
  }
  BatchReq r;
  r.src = src; r.len = len; r.files = files; r.data_digests = data_digests; r.with_data = with_data;
  r.crc_which = crc_which; r.crc_out = crc_out; r.sum_which = sum_which; r.sums = sums;
  // page-locked buffers (mec_alloc_pinned*, or anything cudaHostRegister'ed) are moved by the gather / scatter kernels; checked here,
  // on the caller's thread, so the worker does not pay for it
  r.mapped = mec_is_pinned(src) && (!data_digests || mec_is_pinned(data_digests));
  for (int i = 0; i < b->codec->n && r.mapped; i++)
    if (files[i] && (i >= b->codec->k || with_data)) r.mapped = mec_is_pinned(files[i]) != 0;
  return batcher_enqueue_wait(b, r);
}
extern "C" int64_t mec_batcher_encode(mec_batcher* b, const uint8_t* src, int64_t len, uint8_t* const* files, int write_quorum) {
  return batcher_call(b, src, len, files, nullptr, true, write_quorum);
}
extern "C" int64_t mec_batcher_encode_sg(mec_batcher* b, const uint8_t* src, int64_t len, uint8_t* const* files, uint8_t* data_digests,
                                         int write_quorum) {
  if (!data_digests) return MEC_ERR_INVALID_ARGUMENT;
  return batcher_call(b, src, len, files, data_digests, false, write_quorum);
}
extern "C" int64_t mec_batcher_encode_crc(mec_batcher* b, const uint8_t* src, int64_t len, uint8_t* const* files, uint8_t* data_digests,
                                          int write_quorum, int which, uint64_t* out3) {
  which &= 7;
  if (which && !out3) return MEC_ERR_INVALID_ARGUMENT;
  return batcher_call(b, src, len, files, data_digests, data_digests == nullptr, write_quorum, which, out3);
}
extern "C" int64_t mec_batcher_encode_sums(mec_batcher* b, const uint8_t* src, int64_t len, uint8_t* const* files, uint8_t* data_digests,
                                           int write_quorum, int which, uint64_t* crc3, uint8_t* sums) {
  constexpr int kCrcMask = MEC_CRC32 | MEC_CRC32C | MEC_CRC64NVME;
  if (which & ~(kCrcMask | kSumMask)) return MEC_ERR_INVALID_ARGUMENT;
  if (((which & kCrcMask) && !crc3) || ((which & kSumMask) && !sums)) return MEC_ERR_INVALID_ARGUMENT;
  return batcher_call(b, src, len, files, data_digests, data_digests == nullptr, write_quorum, which & kCrcMask, crc3, which & kSumMask,
                      sums);
}
// The k readers parallelReader picks for a read or move (choose_readers on r.gfiles, r.prefer), chosen on the caller's thread: equal
// reader sets share a batch.  Sets their bits in r.alive_mask and clears *mapped unless every one of them is page-locked.
static int batch_readers(const mec_codec* c, BatchReq& r, bool* mapped) {
  uint8_t alive[kBatchMaxFiles];
  int chosen[kBatchMaxFiles];
  for (int i = 0; i < c->n; i++) alive[i] = r.gfiles[i] != nullptr;
  if (choose_readers(c, r.gfiles, alive, r.prefer, chosen) < c->k) return MEC_ERR_READ_QUORUM;
  for (int t = 0; t < c->k; t++) {
    r.alive_mask |= 1ull << chosen[t];
    *mapped = *mapped && mec_is_pinned(r.gfiles[chosen[t]]) != 0;
  }
  return MEC_OK;
}

// A GET request `r` (files, range, dst and prefer set) into a merged batch, or on its own through the private handle when its buffers
// are not page-locked: the reader set it merges on is chosen here, on the caller's thread.
static int64_t batcher_get(mec_batcher* b, BatchReq& r) {
  const int n = b->codec->n, k = b->codec->k;
  const uint8_t* const* files = r.gfiles;
  bool mapped = !b->sw.memcpy && n <= kBatchMaxFiles && n <= 64 && k <= 32 && mec_is_pinned(r.dst) != 0;
  if (r.prefer && n <= kBatchMaxFiles) {
    // with preferReaders (cmd/erasure-decode.go:92-123): a k-bit mask equals an alive mask only when exactly those k drives are online
    const int rc = batch_readers(b->codec, r, &mapped);
    if (rc) return rc;
  } else {
    int online = 0;
    for (int i = 0; i < n; i++) {
      if (!files[i]) continue;
      online++;
      if (i < 64) r.alive_mask |= 1ull << i;
    }
    if (online < k) return MEC_ERR_READ_QUORUM;
    // only the k readers that will be used have to be mapped
    for (int i = 0, cnt = 0; i < n && cnt < k && mapped; i++)
      if (files[i]) { mapped = mec_is_pinned(files[i]) != 0; cnt++; }
  }
  return mapped ? batcher_enqueue_wait(b, r) : batcher_run_alone(b, r);
}

// Erasure.Decode through the coalescer: GETs that are queued together and read the same drives are merged into one launch — without
// `prefer` the same drives online, with it the same k readers parallelReader picks; with MEC_BATCHER_MIX_PATTERNS any reads.
// Calls whose buffers are not page-locked, and calls that meet bitrot, run on their own through a private handle.
extern "C" int64_t mec_batcher_decode_prefer(mec_batcher* b, const uint8_t* const* files, const uint8_t* prefer, int64_t offset,
                                             int64_t length, int64_t total, uint8_t* dst, int* heal_hint) {
  if (heal_hint) *heal_hint = 0;
  if (!b || !files) return MEC_ERR_INVALID_ARGUMENT;
  if (offset < 0 || length < 0 || offset + length > total) return MEC_ERR_INVALID_ARGUMENT;  // cmd/erasure-decode.go:240-245
  if (length == 0) return 0;
  if (!dst) return MEC_ERR_INVALID_ARGUMENT;
  BatchReq r;
  r.kind = ReqKind::Get; r.gfiles = files; r.offset = offset; r.length = length; r.total = total; r.dst = dst; r.heal_hint = heal_hint;
  r.prefer = prefer;
  return batcher_get(b, r);
}
extern "C" int64_t mec_batcher_decode(mec_batcher* b, const uint8_t* const* files, int64_t offset, int64_t length, int64_t total,
                                      uint8_t* dst, int* heal_hint) {
  return mec_batcher_decode_prefer(b, files, nullptr, offset, length, total, dst, heal_hint);
}

// Erasure.Heal (cmd/erasure-decode.go:317) through the coalescer: heals queued together that read the same k drives and rebuild the
// same stale drives are merged into one fused launch.  Calls the merged path cannot take (pageable buffers, a drive that is both a
// reader and stale, more drives than the kernels' tables hold) and calls that meet bitrot run on their own through mec_heal_prefer
// on a private handle.
extern "C" int mec_batcher_heal(mec_batcher* b, const uint8_t* const* files, const uint8_t* prefer, int64_t total,
                                uint8_t* const* out_files, uint8_t* corrupt) {
  if (!b || !files || !out_files) return MEC_ERR_INVALID_ARGUMENT;
  const int n = b->codec->n;
  BatchReq r;
  r.kind = ReqKind::Heal; r.gfiles = files; r.offset = 0; r.length = total; r.total = total;
  r.prefer = prefer; r.outs = out_files; r.corrupt = corrupt;
  if (n > kBatchMaxFiles || n > 64) return static_cast<int>(batcher_run_alone(b, r));
  if (corrupt) memset(corrupt, 0, static_cast<size_t>(n));
  if (total <= 0) return MEC_OK;
  bool mapped = !b->sw.memcpy;
  const int rc = batch_readers(b->codec, r, &mapped);
  if (rc) return rc;
  int nstale = 0;
  for (int i = 0; i < n; i++)
    if (out_files[i]) {
      r.stale_mask |= 1ull << i;
      nstale++;
      mapped = mapped && mec_is_pinned(out_files[i]) != 0;
    }
  // a drive that is read and also rewritten is passed through unchanged by reconstruct_range: the serial path does that
  if (!mapped || (r.alive_mask & r.stale_mask) != 0 || nstale > kMaxR) return static_cast<int>(batcher_run_alone(b, r));
  return static_cast<int>(batcher_enqueue_wait(b, r));
}

// mec_transcode through the coalescer: moves queued together that read the same k drives (any, with MEC_BATCHER_MIX_PATTERNS) are
// merged into one batch.  Moves the merged path cannot take (pageable buffers, more drives than the kernels' tables hold, parts of
// more than max_batch_blocks blocks, which mec_transcode pipelines over its slots anyway) and moves that meet bitrot run on their own
// through mec_transcode on the private pair.
extern "C" int64_t mec_batcher_transcode(mec_batcher* b, const uint8_t* const* files, const uint8_t* prefer, int64_t total,
                                         uint8_t* const* out_files, int write_quorum, int* heal_hint) {
  if (heal_hint) *heal_hint = 0;
  if (!b || !b->dst || !files || !out_files || total < 0) return MEC_ERR_INVALID_ARGUMENT;
  mec_codec* c = b->codec;
  mec_codec* e = b->dst;
  int online = 0;
  for (int i = 0; i < e->n; i++) online += out_files[i] != nullptr;
  if (online < write_quorum) return MEC_ERR_WRITE_QUORUM;  // cmd/erasure-encode.go:59-65
  if (total == 0) return 0;
  BatchReq r;
  r.kind = ReqKind::Transcode; r.gfiles = files; r.offset = 0; r.length = total; r.total = total;
  r.prefer = prefer; r.heal_hint = heal_hint;
  r.len = total; r.files = out_files; r.with_data = true;  // the destination side, a PUT of the part
  if (c->n > kBatchMaxFiles || e->n > kBatchMaxFiles) return batcher_run_alone(b, r);
  bool mapped = !b->sw.memcpy;
  const int rc = batch_readers(c, r, &mapped);
  if (rc) return rc;
  for (int i = 0; i < e->n && mapped; i++)
    if (out_files[i]) mapped = mec_is_pinned(out_files[i]) != 0;
  if (!mapped || ceil_frac(total, c->block_size) > b->max_blocks) return batcher_run_alone(b, r);
  return batcher_enqueue_wait(b, r);
}

// mec_transcode_whole through the coalescer: whole-file moves of one algorithm queued together that read the same k drives (any,
// with MEC_BATCHER_MIX_PATTERNS) are merged into one batch, staged in one batched copy and hashed in one launch (batch_whole_stage),
// then rebuilt, re-split, encoded and scattered as a batch of streaming moves.  The private path is mec_batcher_transcode's, through
// mec_transcode_whole on a private pair whose source handle carries the request's algorithm.
extern "C" int64_t mec_batcher_transcode_whole(mec_batcher* b, int algo, const uint8_t* const* files, const uint8_t* sums,
                                               const uint8_t* prefer, int64_t total, uint8_t* const* out_files, int write_quorum,
                                               int* heal_hint) {
  if (heal_hint) *heal_hint = 0;
  if (!b || !b->dst || !files || !sums || !out_files || total < 0 || mec_digest_size(algo) < 0) return MEC_ERR_INVALID_ARGUMENT;
  if (algo == MEC_HIGHWAYHASH256S) return MEC_ERR_UNSUPPORTED;  // a streaming part moves through mec_batcher_transcode
  mec_codec* c = b->codec;
  mec_codec* e = b->dst;
  int online = 0;
  for (int i = 0; i < e->n; i++) online += out_files[i] != nullptr;
  if (online < write_quorum) return MEC_ERR_WRITE_QUORUM;  // cmd/erasure-encode.go:59-65
  if (total == 0) return 0;
  BatchReq r;
  r.kind = ReqKind::TranscodeWhole; r.gfiles = files; r.offset = 0; r.length = total; r.total = total;
  r.prefer = prefer; r.heal_hint = heal_hint; r.whole_algo = algo; r.whole_sums = sums;
  r.len = total; r.files = out_files; r.with_data = true;  // the destination side, a PUT of the part
  if (c->n > kBatchMaxFiles || e->n > kBatchMaxFiles) return batcher_run_alone(b, r);
  bool mapped = !b->sw.memcpy;
  const int rc = batch_readers(c, r, &mapped);
  if (rc) return rc;
  r.whole_drives = r.alive_mask;  // every reader is whole-file
  for (int i = 0; i < e->n && mapped; i++)
    if (out_files[i]) mapped = mec_is_pinned(out_files[i]) != 0;
  if (!mapped || ceil_frac(total, c->block_size) > b->max_blocks) return batcher_run_alone(b, r);
  return batcher_enqueue_wait(b, r);
}

// The k readers of a mixed read (mec_batcher_decode_mixed / _heal_mixed), chosen on the caller's thread exactly as mec_decode_mixed /
// mec_heal_mixed choose them: drives with alive[i] set, `prefer` first, then index order.  Sets r.whole_drives (the chosen readers
// that are whole-file) and r.whole_algo (`walgo` when there is one, else 0), and clears *mapped unless every chosen reader is
// page-locked.  Returns the chosen readers' mask, or 0 when fewer than k are alive (MEC_ERR_READ_QUORUM).
static uint64_t mixed_readers(const mec_codec* c, BatchReq& r, const uint8_t* alive, int walgo, bool* mapped) {
  int chosen[kBatchMaxFiles];
  if (choose_readers(c, r.gfiles, alive, r.prefer, chosen) < c->k) return 0;
  uint64_t mask = 0;
  for (int t = 0; t < c->k; t++) {
    const int i = chosen[t];
    mask |= 1ull << i;
    if (r.algos[i] != MEC_HIGHWAYHASH256S) r.whole_drives |= 1ull << i;
    *mapped = *mapped && mec_is_pinned(r.gfiles[i]) != 0;
  }
  r.whole_algo = r.whole_drives ? walgo : 0;
  return mask;
}

// mec_decode_mixed through the coalescer.  A GET whose k chosen readers all stream is an ordinary merged GET (the reader-set rules of
// mec_batcher_decode_prefer); one with a whole-file reader among them joins batches of GETs of the same whole-file algorithm, whose
// whole-file readers are staged whole and hashed in one launch (batch_whole_stage).  Either is redone through mec_decode_mixed on
// the private handle when it meets bitrot.
extern "C" int64_t mec_batcher_decode_mixed(mec_batcher* b, const int* algos, const uint8_t* const* files, const uint8_t* sums,
                                            const uint8_t* prefer, int64_t offset, int64_t length, int64_t total, uint8_t* dst,
                                            int* heal_hint) {
  if (heal_hint) *heal_hint = 0;
  if (!b || !algos || !files) return MEC_ERR_INVALID_ARGUMENT;
  if (offset < 0 || length < 0) return MEC_ERR_INVALID_ARGUMENT;  // cmd/erasure-decode.go:240-242
  if (offset + length > total) return MEC_ERR_INVALID_ARGUMENT;   // :243-245
  if (length == 0) return 0;                                      // :247-249
  if (!dst) return MEC_ERR_INVALID_ARGUMENT;
  mec_codec* c = b->codec;
  int walgo = 0;
  int rc = mixed_formats(c, algos, files, nullptr, sums, &walgo);
  if (rc) return rc;
  const int n = c->n, k = c->k;
  const ReadRange rr = read_range(c, offset, length, total);
  if (static_cast<int64_t>(k) * rr.last_len < std::min(offset + length, total) - rr.last_block * c->block_size) return MEC_ERR_SHORT_DATA;
  BatchReq r;
  r.kind = ReqKind::Get; r.gfiles = files; r.offset = offset; r.length = length; r.total = total; r.dst = dst; r.heal_hint = heal_hint;
  r.prefer = prefer; r.algos = algos; r.whole_sums = sums;
  if (n > kBatchMaxFiles) return batcher_run_alone(b, r);
  uint8_t alive[kBatchMaxFiles];
  for (int i = 0; i < n; i++) alive[i] = files[i] != nullptr;
  bool mapped = !b->sw.memcpy && mec_is_pinned(dst) != 0;
  const uint64_t chosen = mixed_readers(c, r, alive, walgo, &mapped);
  if (!chosen) return MEC_ERR_READ_QUORUM;
  // the reader set batcher_main merges on: as mec_batcher_decode_prefer keys a streaming GET (the drives online without `prefer`),
  // the chosen readers for a GET with a whole-file reader
  if (prefer || r.whole_algo) {
    r.alive_mask = chosen;
  } else {
    for (int i = 0; i < n; i++)
      if (files[i]) r.alive_mask |= 1ull << i;
  }
  if (!mapped || (r.whole_algo && ceil_frac(total, c->block_size) > b->max_blocks)) return batcher_run_alone(b, r);
  return batcher_enqueue_wait(b, r);
}

// mec_heal_mixed through the coalescer: as mec_batcher_decode_mixed, with mec_batcher_heal's rules for heals whose k chosen readers
// all stream (the same readers and stale drives share a launch) and mec_heal_mixed as the private path.
extern "C" int mec_batcher_heal_mixed(mec_batcher* b, const int* algos, const uint8_t* const* files, const uint8_t* sums,
                                      const uint8_t* prefer, int64_t total, uint8_t* const* out_files, uint8_t* corrupt) {
  if (!b || !algos || !files || !out_files) return MEC_ERR_INVALID_ARGUMENT;
  mec_codec* c = b->codec;
  const int n = c->n;
  if (corrupt) memset(corrupt, 0, static_cast<size_t>(n));
  int walgo = 0;
  int rc = mixed_formats(c, algos, files, out_files, sums, &walgo);
  if (rc) return rc;
  if (total <= 0) return MEC_OK;
  BatchReq r;
  r.kind = ReqKind::Heal; r.gfiles = files; r.offset = 0; r.length = total; r.total = total;
  r.prefer = prefer; r.outs = out_files; r.corrupt = corrupt; r.algos = algos; r.whole_sums = sums;
  if (n > kBatchMaxFiles) return static_cast<int>(batcher_run_alone(b, r));
  // healObject opens no reader on a drive it heals (cmd/erasure-healing.go:572-575): a stale drive is never read
  uint8_t alive[kBatchMaxFiles];
  for (int i = 0; i < n; i++) alive[i] = files[i] != nullptr && out_files[i] == nullptr;
  bool mapped = !b->sw.memcpy;
  r.alive_mask = mixed_readers(c, r, alive, walgo, &mapped);
  if (!r.alive_mask) return MEC_ERR_READ_QUORUM;
  int nstale = 0;
  for (int i = 0; i < n; i++)
    if (out_files[i]) {
      r.stale_mask |= 1ull << i;
      nstale++;
      mapped = mapped && mec_is_pinned(out_files[i]) != 0;
    }
  if (!mapped || nstale > kMaxR || (r.whole_algo && ceil_frac(total, c->block_size) > b->max_blocks))
    return static_cast<int>(batcher_run_alone(b, r));
  return static_cast<int>(batcher_enqueue_wait(b, r));
}

// The staged bytes of a verify call whose parts are decided (verify_decide): a frame pitch per streaming frame, a 16-byte-aligned file
// and 256 bytes behind it per whole-file part (batcher_submit_verify's layout).  Clears *mapped unless every file to hash is page-locked.
static int64_t verify_staged(const mec_codec* c, const BatchReq& r, bool* mapped) {
  const int64_t S = c->S(), P = round_up(32 + S, 16);
  int64_t bytes = 0;
  for (int64_t p = 0; p < r.vparts; p++) {
    if (r.vresults[p] != MEC_OK) continue;
    const bool streaming = r.valgos[p] == MEC_HIGHWAYHASH256S;
    bytes += streaming ? ceil_frac(r.vpart_lens[p], S) * P : round_up(r.vfile_lens[p], 16) + 256;
    if (r.vfile_lens[p] > 0) *mapped = *mapped && mec_is_pinned(r.vfiles[p]) != 0;
  }
  return bytes;
}

// VerifyFile (cmd/xl-storage.go:3100-3137) through the coalescer: mec_bitrot_verify_parts on the batcher's geometry.  Refusals and the
// per-part decisions that need no device are made on the caller's thread; the parts left to hash join a merged verify batch
// (batcher_submit_verify), or run through mec_bitrot_verify_parts on the private handle when the call cannot ride in one.
extern "C" int mec_batcher_verify(mec_batcher* b, int64_t nparts, const int* algos, const uint8_t* const* files, const int64_t* file_lens,
                                  const int64_t* part_lens, const uint8_t* sums, int* results) {
  NvtxRange nvtx("mec_batcher_verify");
  if (!b || !verify_args_ok(nparts, algos, files, file_lens, part_lens, sums, results)) return MEC_ERR_INVALID_ARGUMENT;
  mec_codec* c = b->codec;
  BatchReq r;
  r.kind = ReqKind::Verify;
  verify_decide(c->S(), nparts, algos, files, file_lens, part_lens, results, &r.vframes, &r.vwhole);
  if (r.vframes == 0 && r.vwhole == 0) return MEC_OK;
  r.vparts = nparts; r.valgos = algos; r.vfiles = files; r.vfile_lens = file_lens; r.vpart_lens = part_lens; r.vsums = sums;
  r.vresults = results;
  bool mapped = !b->sw.memcpy;
  r.vbytes = verify_staged(c, r, &mapped);
  const VerifyLimits lim = verify_limits(b);
  if (!mapped || r.vframes > lim.frames || r.vbytes > lim.bytes || r.vwhole > lim.files) {
    b->st_verifies_serial++;
    mec_codec* sc = batcher_private(b, c, b->serial);
    return sc ? mec_bitrot_verify_parts(sc, nparts, algos, files, file_lens, part_lens, sums, results) : MEC_ERR_UNEXPECTED;
  }
  return static_cast<int>(batcher_enqueue_wait(b, r));
}

// EncryptRequest + Erasure.Encode through the coalescer: mec_encode_sse's refusals on the caller's thread, then the request joins a
// merged PUT batch as its ciphertext of mec_dare_encrypted_size(len) bytes; the batch seals it (sse_put_plan, sse_put_seal).  Calls
// whose buffers are not page-locked, and MEC_BATCHER_MEMCPY, go through mec_encode_sse on the private handle.
extern "C" int64_t mec_batcher_encode_sse(mec_batcher* b, const uint8_t* src, int64_t len, const uint8_t* key, const uint8_t* nonce,
                                          uint8_t* const* files, int write_quorum) {
  NvtxRange nvtx("mec_batcher_encode_sse");
  if (!b || len < 0 || !files || !key || !nonce || (len > 0 && !src)) return MEC_ERR_INVALID_ARGUMENT;
  const int64_t E = mec_dare_encrypted_size(len);
  if (E < 0) return E;
  const int n = b->codec->n;
  int online = 0;
  for (int i = 0; i < n; i++) online += files[i] != nullptr;
  if (online < write_quorum) return MEC_ERR_WRITE_QUORUM;  // cmd/erasure-encode.go:59-65
  if (len == 0) return 0;
  BatchReq r;
  r.src = src; r.len = E; r.files = files; r.with_data = true;
  r.sse_key = key; r.sse_nonce = nonce; r.sse_len = len; r.sse_chacha = b->dare_chacha20.load();
  bool mapped = !b->sw.memcpy && mec_is_pinned(src) != 0;
  for (int i = 0; i < n && mapped; i++)
    if (files[i]) mapped = mec_is_pinned(files[i]) != 0;
  r.mapped = mapped;
  return mapped ? batcher_enqueue_wait(b, r) : batcher_run_alone(b, r);
}

// Erasure.Decode + DecryptBlocksRequestR through the coalescer, one part per call: mec_decode_sse's refusals on the caller's thread,
// then the ciphertext range of the whole packages that hold [offset, offset + length) is read as an ordinary merged GET (the reader
// rules of mec_batcher_decode_prefer) and opened by the batch (sse_get_open).  A request that meets bitrot is redone alone through
// mec_decode_sse on the private handle, as are calls whose buffers are not page-locked.
extern "C" int64_t mec_batcher_decode_sse(mec_batcher* b, const uint8_t* const* files, const uint8_t* prefer, int64_t offset,
                                          int64_t length, int64_t enc_total, const uint8_t* key, uint8_t* dst, int* heal_hint) {
  NvtxRange nvtx("mec_batcher_decode_sse");
  if (heal_hint) *heal_hint = 0;
  if (!b || !files || !key || offset < 0 || length < 0 || enc_total < 0) return MEC_ERR_INVALID_ARGUMENT;
  const int64_t D = mec_dare_decrypted_size(enc_total);
  if (D < 0) return MEC_ERR_NOT_AUTHENTIC;  // ObjectInfo.DecryptedSize: errObjectTampered
  if (offset + length > D) return MEC_ERR_INVALID_ARGUMENT;
  if (length == 0) return 0;
  if (!dst) return MEC_ERR_INVALID_ARGUMENT;
  const mec_codec* c = b->codec;
  const int64_t p_first = offset / kPkg, p_last = (offset + length - 1) / kPkg;
  const int64_t eoff = p_first * kEPkg, eend = std::min(enc_total, (p_last + 1) * kEPkg);
  const ReadRange rr = read_range(c, eoff, eend - eoff, enc_total);
  if (static_cast<int64_t>(c->k) * rr.last_len < eend - rr.last_block * c->block_size) return MEC_ERR_SHORT_DATA;  // as mec_decode_sse
  BatchReq r;
  r.kind = ReqKind::Get; r.gfiles = files; r.offset = eoff; r.length = eend - eoff; r.total = enc_total; r.dst = dst;
  r.heal_hint = heal_hint; r.prefer = prefer;
  r.sse_key = key; r.sse_offset = offset; r.sse_len = length; r.sse_total = D; r.sse_chacha = b->dare_chacha20.load();
  return batcher_get(b, r);
}

// Options of a batcher: "dare_chacha20" (0, 1, 2; see mec_set_option) for its codec and private handle.  Each encrypted request
// records the value when it is admitted and runs under it, whichever batch it merges into and if it is redone alone.
extern "C" int mec_batcher_set_option(mec_batcher* b, const char* name, int64_t value) {
  if (!b || !name || strcmp(name, "dare_chacha20") != 0 || value < 0 || value > 2) return MEC_ERR_INVALID_ARGUMENT;
  std::lock_guard<std::mutex> lk(b->serial_mu);  // a private handle created meanwhile takes the new value
  b->dare_chacha20 = static_cast<int>(value);
  int rc = mec_set_option(b->codec, name, value);
  if (rc == MEC_OK && b->serial) rc = mec_set_option(b->serial, name, value);
  return rc;
}

extern "C" int64_t mec_batcher_stat(const mec_batcher* b, const char* name) {
  if (!b || !name) return -1;
  if (!strcmp(name, "batches")) return b->st_batches.load();
  if (!strcmp(name, "requests")) return b->st_requests.load();
  if (!strcmp(name, "blocks")) return b->st_blocks.load();
  if (!strcmp(name, "kernel_batches")) return b->st_kernel_batches.load();
  if (!strcmp(name, "redone")) return b->st_redone.load();
  if (!strcmp(name, "crc_requests")) return b->st_crc_requests.load();
  if (!strcmp(name, "sum_requests")) return b->st_sum_requests.load();
  if (!strcmp(name, "patterns")) return b->st_patterns.load();
  if (!strcmp(name, "mixed_batches")) return b->st_mixed.load();
  if (!strcmp(name, "launches")) return b->codec->eng ? b->codec->eng->launches() : 0;
  if (!strcmp(name, "us_submit")) return b->us_submit.load();
  if (!strcmp(name, "us_sync")) return b->us_sync.load();
  if (!strcmp(name, "us_finish")) return b->us_finish.load();
  if (!strcmp(name, "us_idle")) return b->us_idle.load();
  if (!strcmp(name, "us_stage")) return b->us_stage.load();
  if (!strcmp(name, "us_kernel")) return b->us_kernel.load();
  if (!strcmp(name, "us_scatter")) return b->us_scatter.load();
  if (!strcmp(name, "transcodes")) return b->st_transcodes.load();
  if (!strcmp(name, "transcodes_serial")) return b->st_transcodes_serial.load();
  if (!strcmp(name, "transcodes_whole")) return b->st_transcodes_whole.load();
  if (!strcmp(name, "transcodes_whole_serial")) return b->st_transcodes_whole_serial.load();
  if (!strcmp(name, "reads_whole")) return b->st_reads_whole.load();
  if (!strcmp(name, "reads_whole_serial")) return b->st_reads_whole_serial.load();
  if (!strcmp(name, "verifies")) return b->st_verifies.load();
  if (!strcmp(name, "verifies_serial")) return b->st_verifies_serial.load();
  if (!strcmp(name, "sse_puts")) return b->st_sse_puts.load();
  if (!strcmp(name, "sse_gets")) return b->st_sse_gets.load();
  if (!strcmp(name, "sse_serial")) return b->st_sse_serial.load();
  if (!strncmp(name, "dst_", 4)) return b->dst ? mec_get_stat(b->dst, name + 4) : -1;  // the destination codec of merged moves
  return mec_get_stat(b->codec, name);  // the batcher's codec: which kernel forms its merged launches ran ("form_*", "last_*", ...)
}
