// ec_engine.cu — kernel instantiation + dispatch for the fused RS + HighwayHash kernel.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <dlfcn.h>
#include <sys/stat.h>
#include <unistd.h>
#include <atomic>
#include <nvrtc.h>
#include <chrono>
#include <condition_variable>
#include <deque>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <vector>
#include "../../include/minio_ec.h"
#include "ec_engine.h"
#include "ec_small.cuh"
#include "jit_headers.inc"

namespace mec {

static thread_local std::string g_last_error;
void set_last_error(const std::string& s) { g_last_error = s; }
const char* get_last_error() { return g_last_error.c_str(); }

int DevBuf::ensure(size_t n) {
  if (n <= cap) return MEC_OK;
  release();
  size_t want = n + (n >> 3) + 256;
  MEC_CUDA_OK(cudaMalloc(&p, want));
  cap = want;
  return MEC_OK;
}
void DevBuf::release() {
  if (p) cudaFree(p);
  p = nullptr;
  cap = 0;
}

// (k, m) pairs with compile-time specialised GF code.  MinIO's default parity for a 16-drive set
// is EC:4 => RS(12,4) (internal/config/storageclass/storage-class.go:355); the others are the
// BASELINE configs and common set sizes.
// X(K, M, S mod 16 for 1 MiB blocks)
#define MEC_STATIC_CONFIGS(X) X(12, 4, 6) X(4, 2, 0) X(16, 4, 0) X(8, 8, 0) X(8, 4, 0) X(6, 2, 11) X(2, 2, 0)

using KernelFn = void (*)(const FusedParams, const TmaMaps);
using SmallFn = void (*)(const FusedParams);  // latency kernel (ec_small.cuh): one erasure block per CTA
constexpr int kStaticEb = 4;  // erasure blocks per CTA of the compile-time specialised kernels
// raw-tile bytes in flight per SM that the 3-D-fetch encode of misaligned rows is sized to (launch_fused): five RS(12,4) CTAs
constexpr int64_t kRawBytesInFlightPerSm = 5 * 12 * 1152;

struct StaticEntry {
  int k, m, sm16;
  KernelFn fast3d;    // TMA, S mod 16 == sm16, eb == kStaticEb, one 3-D request per tile
  KernelFn fast3d_auto;  // same, warp-autonomous pipeline (k + m == 16 and misaligned rows only), else nullptr
  KernelFn fast3d_semi;  // same, barrier (B) warp-local
  KernelFn fast_auto, aligned_auto;  // warp-autonomous pipeline (k + m == 16 only), else nullptr
  KernelFn fast;      // TMA, S mod 16 == sm16, eb == kStaticEb
  KernelFn aligned;   // TMA, S mod 16 == 0,    eb == kStaticEb
  KernelFn runtime;   // TMA, any alignment (per-row table), runtime eb
  KernelFn bytewise;  // byte-wise loader, runtime eb
  SmallFn small;      // latency kernel for launches that cannot fill the GPU
};
static const StaticEntry kStaticTable[] = {
#define X(K, M, A)                                                                                      \
  {K, M, A, fused_rs_hh_kernel<GfStatic<K, M>, true, A, kStaticEb, 0, true>,                          \
   (K + M == 16 && A != 0) ? fused_rs_hh_kernel<GfStatic<K, M>, true, A, kStaticEb, (K + M == 16 && A != 0) ? 1 : 0, true> : nullptr, \
   (K + M == 16 && A != 0) ? fused_rs_hh_kernel<GfStatic<K, M>, true, A, kStaticEb, (K + M == 16 && A != 0) ? 2 : 0, true> : nullptr, \
   (K + M == 16) ? fused_rs_hh_kernel<GfStatic<K, M>, true, A, kStaticEb, (K + M == 16) ? 1 : 0> : nullptr, \
   (K + M == 16) ? fused_rs_hh_kernel<GfStatic<K, M>, true, 0, kStaticEb, (K + M == 16) ? 1 : 0> : nullptr,          \
   fused_rs_hh_kernel<GfStatic<K, M>, true, A, kStaticEb, 0>,                                        \
   fused_rs_hh_kernel<GfStatic<K, M>, true, 0, kStaticEb, 0>,                                        \
   fused_rs_hh_kernel<GfStatic<K, M>, true, kAlignRuntime, 0, 0>, fused_rs_hh_kernel<GfStatic<K, M>, false, 0, 0, 0>, \
   small_rs_hh_kernel<GfStatic<K, M>, small_gf_warps(K + M)>},
    MEC_STATIC_CONFIGS(X)
#undef X
};
// runtime-matrix kernels, indexed by row chunk {1, 2, 4}: a single rebuilt shard (the common single-drive
// failure) costs a quarter of the masked XORs of a four-shard rebuild
static const KernelFn kDynAligned[3] = {fused_rs_hh_kernel<GfDynamic<1>, true, 0, 0, 0>, fused_rs_hh_kernel<GfDynamic<2>, true, 0, 0, 0>,
                                        fused_rs_hh_kernel<GfDynamic<4>, true, 0, 0, 0>};
static const KernelFn kDynRuntime[3] = {fused_rs_hh_kernel<GfDynamic<1>, true, kAlignRuntime, 0, 0>,
                                        fused_rs_hh_kernel<GfDynamic<2>, true, kAlignRuntime, 0, 0>,
                                        fused_rs_hh_kernel<GfDynamic<4>, true, kAlignRuntime, 0, 0>};
static const SmallFn kDynSmall[2][3] = {{small_rs_hh_kernel<GfDynamic<1>, 3>, small_rs_hh_kernel<GfDynamic<2>, 3>, small_rs_hh_kernel<GfDynamic<4>, 3>},
                                        {small_rs_hh_kernel<GfDynamic<1>, 4>, small_rs_hh_kernel<GfDynamic<2>, 4>, small_rs_hh_kernel<GfDynamic<4>, 4>}};
static const KernelFn kDynBytewise[3] = {fused_rs_hh_kernel<GfDynamic<1>, false, 0, 0, 0>, fused_rs_hh_kernel<GfDynamic<2>, false, 0, 0, 0>,
                                         fused_rs_hh_kernel<GfDynamic<4>, false, 0, 0, 0>};

#if MEC_PHASE_CYCLES
// cycle-attribution counters of the instrumented build (ec_kernel.cuh PhaseSlot), one set per process on the device that
// first launched; tools/phase_cycles.py reads and clears them between launches through mec_phase_cycles()
constexpr int kPhaseWords = kPhaseHeader + 8 * kPhaseMaxSm;
static unsigned long long* g_phase_dev = nullptr;
static int phase_clear() {
  std::vector<unsigned long long> init(kPhaseWords, 0ull);
  init[0] = ~0ull;  // earliest CTA start: atomicMin
  MEC_CUDA_OK(cudaMemcpy(g_phase_dev, init.data(), kPhaseWords * sizeof(unsigned long long), cudaMemcpyHostToDevice));
  return MEC_OK;
}
static unsigned long long* phase_counters() {
  if (g_phase_dev == nullptr && (cudaMalloc(&g_phase_dev, kPhaseWords * sizeof(unsigned long long)) != cudaSuccess || phase_clear() != MEC_OK)) {
    cudaGetLastError();
    g_phase_dev = nullptr;
  }
  return g_phase_dev;
}
#endif

}  // namespace mec

#if MEC_PHASE_CYCLES
// copies the first min(n, words) counters to `out` (after a device synchronise), then clears them when `clear` is set;
// returns the number of counter words, -1 before the first launch
extern "C" int mec_phase_cycles(unsigned long long* out, int n, int clear) {
  using namespace mec;
  if (g_phase_dev == nullptr) return -1;
  if (cudaDeviceSynchronize() != cudaSuccess) return -1;
  if (out != nullptr && n > 0 &&
      cudaMemcpy(out, g_phase_dev, static_cast<size_t>(n < kPhaseWords ? n : kPhaseWords) * sizeof(unsigned long long), cudaMemcpyDeviceToHost) != cudaSuccess)
    return -1;
  if (clear && phase_clear() != MEC_OK) return -1;
  return kPhaseWords;
}
#endif

namespace mec {

// ------------------------------------------------------------------------------------------------
// Run-time specialisation.  Decode matrices depend on which shards survived, so they cannot be
// compiled ahead of time; the runtime-matrix kernel pays 8·r masked XORs per input word where the
// compile-time path pays ~9 ops per word for all four outputs.  For large launches the kernel
// template is therefore instantiated for the concrete matrix with NVRTC (≈0.8 s, cached per
// (k, r, matrix)) — the GPU analogue of klauspost/reedsolomon caching inverted matrices per pattern.
#define MEC_STR2(x) #x
#define MEC_STR(x) MEC_STR2(x)
struct NvrtcApi {
  void* h = nullptr;
  decltype(&nvrtcCreateProgram) create = nullptr;
  decltype(&nvrtcDestroyProgram) destroy = nullptr;
  decltype(&nvrtcAddNameExpression) add_name = nullptr;
  decltype(&nvrtcCompileProgram) compile = nullptr;
  decltype(&nvrtcGetCUBINSize) cubin_size = nullptr;
  decltype(&nvrtcGetCUBIN) cubin = nullptr;
  decltype(&nvrtcGetLoweredName) lowered = nullptr;
  decltype(&nvrtcGetProgramLogSize) log_size = nullptr;
  decltype(&nvrtcGetProgramLog) log = nullptr;
  bool ok = false;
};
static NvrtcApi load_nvrtc() {
  NvrtcApi api;
  for (const char* name : {"libnvrtc.so.12", "/usr/local/cuda/lib64/libnvrtc.so.12", "libnvrtc.so"}) {
    api.h = dlopen(name, RTLD_NOW | RTLD_LOCAL);
    if (api.h) break;
  }
  if (!api.h) return api;
#define MEC_SYM(field, sym) api.field = reinterpret_cast<decltype(api.field)>(dlsym(api.h, #sym))
  MEC_SYM(create, nvrtcCreateProgram); MEC_SYM(destroy, nvrtcDestroyProgram); MEC_SYM(add_name, nvrtcAddNameExpression);
  MEC_SYM(compile, nvrtcCompileProgram); MEC_SYM(cubin_size, nvrtcGetCUBINSize); MEC_SYM(cubin, nvrtcGetCUBIN);
  MEC_SYM(lowered, nvrtcGetLoweredName); MEC_SYM(log_size, nvrtcGetProgramLogSize); MEC_SYM(log, nvrtcGetProgramLog);
#undef MEC_SYM
  api.ok = api.create && api.destroy && api.add_name && api.compile && api.cubin_size && api.cubin && api.lowered && api.log_size && api.log;
  return api;
}
// reached from the background compiler, from synchronous jit = 1 callers and from mec_jit_compile_check: the function-local
// static is initialised exactly once (thread-safe since C++11), so no caller can see a half-filled table
static NvrtcApi& nvrtc_api() {
  static NvrtcApi api = load_nvrtc();
  return api;
}

// The cache is process-wide (per device): MinIO builds one Erasure per request (cmd/erasure-object.go:1371), so a
// per-codec cache would recompile the same erasure pattern for every object of a heal sweep.
//
// Policy.  A compile costs ≈0.4 s of one host core; the specialised kernel saves ≈0.6 ms per GiB over the generic one, so
// stalling a request for it never pays inside that request.  In automatic mode (option jit = -1) a pattern is therefore
// compiled on a background thread once it has been seen with kJitHeatBytes of input, the requests that arrive meanwhile
// run the generic runtime-matrix kernel, and later requests pick the specialised kernel up from the cache.  jit = 1
// compiles (or waits for the background compile) synchronously — tests and benchmarks; jit = 0 never specialises.
namespace {
constexpr int64_t kJitHeatBytes = 32ll << 20;
enum JitState { kJitAbsent = 0, kJitCompiling, kJitReady, kJitFailed };
struct JitSpec {
  int device, k, r, align, eb_t;
  bool rows3d, hash_out;
  std::vector<uint8_t> coef;
};
struct JitEntry {
  std::string key;
  JitSpec spec;
  int state = kJitAbsent;
  void* kernel = nullptr;
  int64_t heat = 0;
};
struct JitGlobals {
  std::mutex mu;
  std::condition_variable cv_done, cv_work;
  std::vector<std::unique_ptr<JitEntry>> cache;
  std::deque<JitEntry*> queue;
  bool worker_started = false, worker_busy = false, stop = false, atexit_registered = false;
  int64_t compiles = 0;
  double seconds = 0;
};
// Never destroyed: the worker thread is detached and must not outlive its mutex.  Process exit while the worker sits
// idle on its condition variable is harmless; exit DURING a compile is not (libnvrtc's own exit handlers tear LLVM state
// down under the compiling thread), hence mec_shutdown() — called by the host before it exits, and registered with
// atexit() after the first compile as a best effort for hosts that do not.
JitGlobals& jit_globals() {
  static JitGlobals* g = new JitGlobals;
  return *g;
}

void jit_quiesce() {
  JitGlobals& g = jit_globals();
  std::unique_lock<std::mutex> lk(g.mu);
  g.stop = true;
  for (JitEntry* e : g.queue) e->state = kJitAbsent;  // never started: a synchronous caller may still compile them
  g.queue.clear();
  g.cv_done.notify_all();
  g.cv_work.notify_all();
  g.cv_done.wait(lk, [&] { return !g.worker_busy; });
}

// On-disk cache of specialised kernels (option: MEC_JIT_CACHE_DIR, default $HOME/.cache/minio_b200; "off" disables): a cubin per
// (kernel sources, compile options, instantiation, matrix), so that a restarted server — or the next process of a heal sweep —
// loads the kernel of an erasure pattern it has met before in a millisecond instead of recompiling for half a second.  Entries
// are keyed by a 64-bit FNV-1a of everything that goes into the compile; files are written to a temporary name and renamed.
static uint64_t fnv1a(uint64_t h, const void* data, size_t n) {
  const unsigned char* p = static_cast<const unsigned char*>(data);
  for (size_t i = 0; i < n; i++) { h ^= p[i]; h *= 1099511628211ull; }
  return h;
}
static std::string jit_cache_dir() {
  const char* e = getenv("MEC_JIT_CACHE_DIR");
  if (e && !strcmp(e, "off")) return "";
  std::string d;
  if (e && *e) d = e;
  else if (const char* h = getenv("HOME")) d = std::string(h) + "/.cache/minio_b200";
  else return "";
  std::string cur;
  for (size_t i = 0; i <= d.size(); i++) {  // mkdir -p
    if (i == d.size() || d[i] == '/') {
      if (!cur.empty()) mkdir(cur.c_str(), 0700);
    }
    if (i < d.size()) cur += d[i];
  }
  return d;
}
static bool read_file(const std::string& path, std::vector<char>* out) {
  FILE* f = fopen(path.c_str(), "rb");
  if (!f) return false;
  fseek(f, 0, SEEK_END);
  const long n = ftell(f);
  fseek(f, 0, SEEK_SET);
  bool ok = n > 0;
  if (ok) {
    out->resize(static_cast<size_t>(n));
    ok = fread(out->data(), 1, static_cast<size_t>(n), f) == static_cast<size_t>(n);
  }
  fclose(f);
  return ok;
}
static void write_file_atomic(const std::string& path, const void* data, size_t n) {
  const std::string tmp = path + ".tmp" + std::to_string(static_cast<long long>(getpid()));
  FILE* f = fopen(tmp.c_str(), "wb");
  if (!f) return;
  const bool ok = fwrite(data, 1, n, f) == n;
  fclose(f);
  if (ok) rename(tmp.c_str(), path.c_str());
  else remove(tmp.c_str());
}

// NVRTC-instantiate the kernel template for one concrete matrix; returns a cudaKernel_t or nullptr
// load == false stops after NVRTC (no device needed): the CPU-side check that the embedded headers still specialise
static std::atomic<int64_t>& jit_cache_hits() {
  static std::atomic<int64_t> n{0};
  return n;
}
void* compile_specialised(const JitSpec& sp, bool load = true) {
  NvrtcApi& api = nvrtc_api();
  if (!api.ok) return nullptr;
  if (load && cudaSetDevice(sp.device) != cudaSuccess) { cudaGetLastError(); return nullptr; }
  const int k = sp.k, r = sp.r;
  void* result = nullptr;
  std::string src = "#include \"ec_kernel.cuh\"\nnamespace mec {\nstruct JitMat { static constexpr int K = " + std::to_string(k) +
                    ", R = " + std::to_string(r) + ";\n  __host__ __device__ static constexpr uint8_t coef(int j, int t) {\n    constexpr uint8_t m[R][K] = {";
  for (int j = 0; j < r; j++) {
    src += "{";
    for (int t = 0; t < k; t++) src += std::to_string(sp.coef[static_cast<size_t>(j) * k + t]) + (t + 1 < k ? "," : "");
    src += j + 1 < r ? "}," : "}";
  }
  src += "};\n    return m[j][t]; } };\nstruct GfJit { static constexpr bool kIsStatic = true; static constexpr int K = JitMat::K, R = JitMat::R, kHashOut = " +
         std::string(sp.hash_out ? "1" : "0") + "; using Mat = JitMat; };\n}\n";
  const char* names[] = {"rtc_compat.h", "gf256.h", "ec_device.cuh", "ec_kernel.cuh"};
  const char* bodies[] = {kJitHdr_rtc_compat_h, kJitHdr_gf256_h, kJitHdr_ec_device_cuh, kJitHdr_ec_kernel_cuh};
  nvrtcProgram prog = nullptr;
  const std::string expr_s = "mec::fused_rs_hh_kernel<mec::GfJit, true, " + std::to_string(sp.align) + ", " + std::to_string(sp.eb_t) +
                             ", 0, " + (sp.rows3d ? "true" : "false") + ">";
  const char* expr = expr_s.c_str();
  if (api.create(&prog, src.c_str(), "mec_jit.cu", 4, bodies, names) != NVRTC_SUCCESS) return nullptr;
  api.add_name(prog, expr);
  const char* opts[] = {"--gpu-architecture=sm_90a", "-std=c++17", "-default-device",
                        "-DMEC_HH_MUL=" MEC_STR(MEC_HH_MUL), "-DMEC_HH_VARIANT=" MEC_STR(MEC_HH_VARIANT),
                        "-DMEC_MIN_BLOCKS=" MEC_STR(MEC_MIN_BLOCKS),
                        "-DMEC_GF_LEVEL=" MEC_STR(MEC_GF_LEVEL), "-DMEC_GF_GROUP=" MEC_STR(MEC_GF_GROUP),
                        "-DMEC_PHASE_CYCLES=" MEC_STR(MEC_PHASE_CYCLES)};
  // disk cache: the key covers the embedded headers, the generated source, the instantiation and the options
  std::string cache_path, cached_name;
  if (load) {
    const std::string dir = jit_cache_dir();
    if (!dir.empty()) {
      uint64_t h = 14695981039346656037ull;
      for (const char* b : bodies) h = fnv1a(h, b, strlen(b));
      h = fnv1a(h, src.data(), src.size());
      h = fnv1a(h, expr_s.data(), expr_s.size());
      for (const char* o : opts) h = fnv1a(h, o, strlen(o));
      char name[64];
      snprintf(name, sizeof(name), "/k%016llx.cubin", static_cast<unsigned long long>(h));
      cache_path = dir + name;
      std::vector<char> blob;
      // file = [u32 length of the lowered kernel name][name][cubin]
      if (read_file(cache_path, &blob) && blob.size() > 8) {
        uint32_t nl = 0;
        memcpy(&nl, blob.data(), 4);
        if (nl > 0 && nl < 4096 && blob.size() > 4 + nl) {
          cached_name.assign(blob.data() + 4, nl);
          cudaLibrary_t lib = nullptr;
          cudaKernel_t kern = nullptr;
          if (cudaLibraryLoadData(&lib, blob.data() + 4 + nl, nullptr, nullptr, 0, nullptr, nullptr, 0) == cudaSuccess &&
              cudaLibraryGetKernel(&kern, lib, cached_name.c_str()) == cudaSuccess) {
            api.destroy(&prog);
            jit_cache_hits()++;
            return reinterpret_cast<void*>(kern);
          }
          cudaGetLastError();  // stale or damaged entry: fall through to a fresh compile, which overwrites it
        }
      }
    }
  }
  nvrtcResult rc = api.compile(prog, static_cast<int>(sizeof(opts) / sizeof(opts[0])), opts);
  if (rc == NVRTC_SUCCESS) {
    size_t sz = 0;
    const char* lname = nullptr;
    if (api.cubin_size(prog, &sz) == NVRTC_SUCCESS && sz > 0 && api.lowered(prog, expr, &lname) == NVRTC_SUCCESS) {
      std::vector<char> cubin(sz);
      api.cubin(prog, cubin.data());
      if (!load) {
        api.destroy(&prog);
        return reinterpret_cast<void*>(static_cast<uintptr_t>(sz));  // compiled: cubin size as a non-null token
      }
      cudaLibrary_t lib = nullptr;
      cudaKernel_t kern = nullptr;
      if (cudaLibraryLoadData(&lib, cubin.data(), nullptr, nullptr, 0, nullptr, nullptr, 0) == cudaSuccess &&
          cudaLibraryGetKernel(&kern, lib, lname) == cudaSuccess) {
        result = reinterpret_cast<void*>(kern);
        if (!cache_path.empty()) {
          const uint32_t nl = static_cast<uint32_t>(strlen(lname));
          std::vector<char> blob(4 + nl + sz);
          memcpy(blob.data(), &nl, 4);
          memcpy(blob.data() + 4, lname, nl);
          memcpy(blob.data() + 4 + nl, cubin.data(), sz);
          write_file_atomic(cache_path, blob.data(), blob.size());
        }
      } else {
        cudaGetLastError();
      }
    }
  } else {
    size_t ls = 0;
    api.log_size(prog, &ls);
    std::string log(ls, 0);
    if (ls) api.log(prog, &log[0]);
    set_last_error("NVRTC specialisation failed, using the runtime-matrix kernel: " + log.substr(0, 800));
  }
  api.destroy(&prog);
  return result;
}

// compile `e` (state already kJitCompiling, mutex NOT held), publish the result
void jit_run(JitGlobals& g, JitEntry* e) {
  const auto t0 = std::chrono::steady_clock::now();
  void* kern = compile_specialised(e->spec);
  const double sec = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  {
    std::lock_guard<std::mutex> lk(g.mu);
    e->kernel = kern;
    e->state = kern ? kJitReady : kJitFailed;  // failures are cached too: never retried, the generic kernel serves
    g.compiles++;
    g.seconds += sec;
  }
  g.cv_done.notify_all();
}

void jit_worker_main() {
  JitGlobals& g = jit_globals();
  for (;;) {
    JitEntry* e = nullptr;
    {
      std::unique_lock<std::mutex> lk(g.mu);
      g.cv_work.wait(lk, [&] { return g.stop || !g.queue.empty(); });
      if (g.stop) return;
      e = g.queue.front();
      g.queue.pop_front();
      g.worker_busy = true;
    }
    jit_run(g, e);
    {
      std::lock_guard<std::mutex> lk(g.mu);
      g.worker_busy = false;
      if (!g.atexit_registered) {  // registered late on purpose: runs before the handlers libnvrtc installed while compiling
        g.atexit_registered = true;
        atexit(jit_quiesce);
      }
    }
    g.cv_done.notify_all();
  }
}
}  // namespace

void jit_shutdown() { jit_quiesce(); }

int64_t jit_compile_check(int k, int r, const uint8_t* coef, int align, int eb_t, bool rows3d, bool hash_out) {
  if (!nvrtc_api().ok) return -1;
  JitSpec sp{0, k, r, align, eb_t, rows3d, hash_out, std::vector<uint8_t>(coef, coef + static_cast<size_t>(k) * r)};
  return static_cast<int64_t>(reinterpret_cast<uintptr_t>(compile_specialised(sp, false)));
}

int64_t Engine::jit_compiles() const {
  JitGlobals& g = jit_globals();
  std::lock_guard<std::mutex> lk(g.mu);
  return g.compiles;
}
int64_t Engine::jit_disk_hits() const { return jit_cache_hits().load(); }
double Engine::jit_seconds() const {
  JitGlobals& g = jit_globals();
  std::lock_guard<std::mutex> lk(g.mu);
  return g.seconds;
}

// mode 1: return the specialised kernel, compiling or waiting for it; mode -1: return it if it is ready, otherwise
// account `in_bytes` to the pattern and hand it to the background worker once it is warm.
void* Engine::jit_kernel(int k, int r, const uint8_t* coef, int align, int eb_t, bool rows3d, bool hash_out, int mode,
                         int64_t in_bytes) {
  std::string key(reinterpret_cast<const char*>(coef), static_cast<size_t>(k) * r);
  key = "d" + std::to_string(device_) + ":" + std::to_string(k) + "x" + std::to_string(r) + "a" + std::to_string(align) + "e" +
        std::to_string(eb_t) + (rows3d ? "3" : "2") + (hash_out ? "h" : "n") + ":" + key;
  JitGlobals& g = jit_globals();
  std::unique_lock<std::mutex> lk(g.mu);
  JitEntry* e = nullptr;
  for (auto& c : g.cache)
    if (c->key == key) { e = c.get(); break; }
  if (!e) {
    g.cache.emplace_back(new JitEntry);
    e = g.cache.back().get();
    e->key = key;
    e->spec = JitSpec{device_, k, r, align, eb_t, rows3d, hash_out, std::vector<uint8_t>(coef, coef + static_cast<size_t>(k) * r)};
  }
  if (e->state == kJitReady) return e->kernel;
  if (e->state == kJitFailed) return nullptr;
  if (mode == 1) {
    while (e->state != kJitReady && e->state != kJitFailed) {
      if (e->state == kJitAbsent) {
        e->state = kJitCompiling;
        lk.unlock();
        jit_run(g, e);
        lk.lock();
      } else {
        g.cv_done.wait(lk);  // the background worker (or another caller) is on it
      }
    }
    return e->state == kJitReady ? e->kernel : nullptr;
  }
  e->heat += in_bytes;
  if (e->state == kJitAbsent && e->heat >= kJitHeatBytes && !g.stop) {
    e->state = kJitCompiling;
    g.queue.push_back(e);
    if (!g.worker_started) {
      g.worker_started = true;
      std::thread(jit_worker_main).detach();
    }
    g.cv_work.notify_one();
  }
  return nullptr;
}

Engine::Engine(int device) : device_(device) {}
Engine::~Engine() {
  if (claim_slots_) { cudaSetDevice(device_); cudaFree(claim_slots_); }
}

int Engine::init() {
  int count = 0;
  cudaError_t e = cudaGetDeviceCount(&count);
  if (e != cudaSuccess || count == 0) {
    set_last_error("no CUDA device available; this library has no CPU fallback");
    return MEC_ERR_NO_DEVICE;
  }
  if (device_ < 0 || device_ >= count) return MEC_ERR_INVALID_ARGUMENT;
  MEC_CUDA_OK(cudaSetDevice(device_));
  cudaDeviceProp prop;
  MEC_CUDA_OK(cudaGetDeviceProperties(&prop, device_));
  num_sms_ = prop.multiProcessorCount;
  if (prop.major != 9 || prop.minor != 0) {  // sm_90a code loads on compute capability 9.0 only
    set_last_error("device is not sm_90 (kernels are built for sm_90a only)");
    return MEC_ERR_UNSUPPORTED;
  }
  cudaDriverEntryPointQueryResult qres;
  MEC_CUDA_OK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &encode_tiled_, cudaEnableDefault, &qres));
  if (qres != cudaDriverEntryPointSuccess || !encode_tiled_) {
    set_last_error("cuTensorMapEncodeTiled not available");
    return MEC_ERR_CUDA;
  }
  return MEC_OK;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static int make_map(void* fn, CUtensorMap* map, const void* base, uint64_t dim0, uint64_t dim1, uint64_t stride1,
                    uint32_t box0, uint32_t box1, uint64_t dim2 = 0, uint64_t stride2 = 0, uint32_t box2 = 0) {
  cuuint64_t dims[3] = {dim0, dim1, dim2};
  cuuint64_t strides[2] = {stride1, stride2};
  cuuint32_t box[3] = {box0, box1, box2};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = reinterpret_cast<EncodeTiledFn>(fn)(map, CU_TENSOR_MAP_DATA_TYPE_UINT32, dim2 ? 3 : 2, const_cast<void*>(base),
                                                    dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                                    CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                                                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error("cuTensorMapEncodeTiled failed with CUresult " + std::to_string(static_cast<int>(r)));
    return MEC_ERR_CUDA;
  }
  return MEC_OK;
}

// cudaFuncAttributeMaxDynamicSharedMemorySize is one number per kernel and device, shared by every handle of the process: the
// runtime-matrix kernels are launched with footprints that depend on (k, r), so the limit is only ever raised (setting it for a
// smaller launch would make the next larger one — possibly another handle's — fail with "invalid argument")
int Engine::raise_smem_limit(const void* kfn, size_t smem) {
  struct Entry { int device; const void* fn; size_t smem; };
  static std::mutex mu;
  static std::vector<Entry> limits;
  std::lock_guard<std::mutex> lk(mu);
  for (auto& e : limits)
    if (e.device == device_ && e.fn == kfn) {
      if (e.smem >= smem) return MEC_OK;
      MEC_CUDA_OK(cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
      e.smem = smem;
      return MEC_OK;
    }
  MEC_CUDA_OK(cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
  limits.push_back(Entry{device_, kfn, smem});
  return MEC_OK;
}

int Engine::launch_fused(const FusedDesc& d, const EngineOptions& opt, cudaStream_t st) {
  if (d.nblocks <= 0 || d.S < 0) return MEC_OK;
  if (d.S == 0 && (d.r > 0 || d.digests == nullptr)) return MEC_OK;  // S == 0: digest of the empty message only
  if (d.k <= 0 || d.k > kMaxK || d.r < 0 || d.r > kMaxR) return MEC_ERR_UNSUPPORTED;
  const int n = d.k + d.r;
  if (2 * n > 256) return MEC_ERR_UNSUPPORTED;
  MEC_CUDA_OK(cudaSetDevice(device_));

  FusedParams p;
  memset(&p, 0, sizeof(p));
  TmaMaps maps;
  memset(&maps, 0, sizeof(maps));
  p.k = d.k;
  p.r = d.r;
  p.nblocks = d.nblocks;
  p.S = d.S;
  p.out = d.out;
  p.out_pitch = d.out_pitch;
  p.digests = d.digests;
  p.nhash = d.hash_outputs ? d.k + d.r : d.k;
  p.corrupt = d.corrupt;
  p.expect_block_stride = d.expect_block_stride;
  for (int t = 0; t < d.k; t++) p.expect_ptr[t] = d.expect_ptr[t];
  if (d.key) memcpy(p.key, d.key, 32);
  if (d.r > 0 && (d.out == nullptr || (d.out_pitch & 15) || (reinterpret_cast<uintptr_t>(d.out) & 15) ||
                  d.out_pitch < d.S))
    return MEC_ERR_INVALID_ARGUMENT;

  // ---- erasure blocks per CTA and block size
  int eb = opt.eb > 0 ? opt.eb : (128 / (2 * n) > 0 ? 128 / (2 * n) : 1);
  if (opt.eb <= 0 && d.static_encode && d.contiguous) eb = kStaticEb;  // OOB blocks of a partial group read as zeros
  if (opt.eb <= 0 && !d.contiguous && d.r > 0 && 2 * n * kStaticEb <= 256) eb = kStaticEb;  // reconstruct: the compile-time CTA shape (NVRTC kernels are EB_T = 4)
  if (opt.eb <= 0)  // small launches: shrink the CTA until there are at least ~2 CTAs per SM
    while (eb > 1 && (d.nblocks + eb - 1) / eb < 2ll * num_sms_) eb >>= 1;
  if (false) {}
  else if (eb > d.nblocks) eb = static_cast<int>(d.nblocks);
  while (eb > 1 && 2 * n * eb > 256) eb--;
  if (eb > 255) eb = 255;
  int threads = (2 * n * eb + 31) / 32 * 32;
  p.eb = eb;

  // ---- static / dynamic GF
  const StaticEntry* se = nullptr;
  if (d.static_encode && d.contiguous && d.hash_outputs && !opt.force_dynamic)
    for (const auto& ent : kStaticTable)
      if (ent.k == d.k && ent.m == d.r) se = &ent;
  if (d.block_pattern != nullptr && (se || d.patterns == nullptr)) return MEC_ERR_INVALID_ARGUMENT;
  if (!se && d.block_pattern == nullptr) {
    if (d.r > 0 && d.coef == nullptr) return MEC_ERR_INVALID_ARGUMENT;
    for (int j = 0; j < d.r; j++)
      for (int t = 0; t < d.k; t++) {
        const uint8_t c = d.coef[static_cast<size_t>(j) * d.k + t];
        p.coef[j][t] = c;
      }
  }

  // ---- launches that cannot fill the GPU take the latency kernel: one erasure block per CTA, hash warps decoupled from the GF
  // warps (ec_small.cuh).  The throughput kernel needs ~0.45 ms for a 1 MiB block however few there are (one warp walks it);
  // this one ~0.16 ms up to one block per SM (RS(12,4), H100 80GB HBM3 at a 400 W power limit); a few blocks per SM later both are
  // bound by the same instruction count and the throughput kernel's occupancy wins.
  // Every geometry the engine accepts fits it: otherwise a legal launch would silently fall through to the throughput kernel, and
  // one that only the latency kernel can run (per-block geometry or decode plans) would fail with MEC_ERR_UNSUPPORTED.
  static_assert(small_smem_bytes(kMaxK, kMaxR, true, 4) <= 227 * 1024, "widest latency-kernel launch exceeds shared memory");
  static_assert(32 * small_hash_warps(kMaxK + kMaxR) + 32 * small_gf_warps(kMaxK + kMaxR) <= 256,
                "widest latency-kernel launch exceeds its __launch_bounds__");
  {
    if (small_ok(opt, d.nblocks) && d.S > 0 && (d.contiguous || d.in_ptr[0] != nullptr)) {
      for (int t = 0; t < d.k; t++) p.in_ptr[t] = d.contiguous ? d.in_base + static_cast<int64_t>(t) * d.S : d.in_ptr[t];
      p.in_block_stride = d.in_block_stride;
      p.in_limit = d.contiguous ? d.in_block_len : d.S;
      p.in_shard_step = d.contiguous ? d.S : 0;
      p.block_len = d.block_len;
      p.blocks = d.blocks;
      p.patterns = d.patterns;
      p.block_pattern = d.block_pattern;
      p.tail_block = d.tail_block; p.tail_in_off = d.tail_in_off; p.tail_S = d.tail_S; p.tail_bytes = d.tail_bytes;
      const int gw = small_gf_warps(n);
      const SmallFn sfn = se ? se->small : kDynSmall[gw - 3][d.r <= 1 ? 0 : (d.r == 2 ? 1 : 2)];
      const void* kfn = reinterpret_cast<const void*>(sfn);
      const size_t smem = small_smem_bytes(d.k, d.r, se == nullptr, gw);
      const int threads = 32 * small_hash_warps(n) + 32 * gw;
      if (smem <= 227 * 1024 && threads <= 256) {
        int rc = raise_smem_limit(kfn, smem);
        if (rc) return rc;
        void* args[] = {&p};
        MEC_CUDA_OK(cudaLaunchKernel(kfn, dim3(static_cast<unsigned>(d.nblocks)), dim3(static_cast<unsigned>(threads)), args, smem, st));
        MEC_CUDA_OK(cudaGetLastError());
        launches_++;
        small_launches_++;
        LaunchRecord rec;
        rec.form = kFormSmall;
        rec.eb = 1;
        rec.grid = d.nblocks;
        rec.row_chunk = se ? -1 : (d.r <= 1 ? 0 : (d.r == 2 ? 1 : 2));
        record_launch(rec);
        return MEC_OK;
      }
    }
  }

  // per-block geometry and per-block decode plans exist in the latency kernel only
  if (d.block_len != nullptr || d.blocks != nullptr || d.tail_block >= 0 || d.block_pattern != nullptr) return MEC_ERR_UNSUPPORTED;
  p.tail_block = -1;

  // ---- input addressing + loader choice.  TMA boxes must start on 16-byte boundaries, so each row is
  // fetched from the aligned-down address and the kernel skips in_align[t] bytes.
  const int64_t ntiles = (static_cast<int64_t>(d.S) + kTile - 1) / kTile;
  bool use_tma = !opt.force_bytewise && d.S > 0;
  bool any_misaligned = false, rows3d = false, direct = false;
  int raw_rows = 0;           // rows of the raw tile with the 3-D fetch (raw_rows_3d)
  void* jit3d = nullptr;      // NVRTC-specialised encode kernel with the one-request-per-tile fetch, when it is ready
  bool jit3d_tried = false;
  p.in_block_stride = d.in_block_stride;
  p.raw_pitch = kRawRow;
  if (d.contiguous) {
    p.in_limit = d.in_block_len;
    p.in_shard_step = d.S;
    const int64_t max_c0 = static_cast<int64_t>(d.k) * d.S + ntiles * kTile + 64;
    if ((reinterpret_cast<uintptr_t>(d.in_base) & 15) || (d.in_block_stride & 15) || (d.in_block_len & 15) ||
        max_c0 >= (1ll << 31) || d.nblocks >= (1ll << 31) || (d.nblocks > 1 && d.in_block_stride < d.in_block_len))
      use_tma = false;
    for (int t = 0; t < d.k; t++) {
      const int64_t off = static_cast<int64_t>(t) * d.S;
      p.in_ptr[t] = d.in_base + off;
      p.in_c0[t] = static_cast<int32_t>(off & ~15ll);
      p.in_align[t] = static_cast<uint8_t>(off & 15);
      any_misaligned |= (off & 15) != 0;
    }
    // every row 16-byte aligned and a kernel instantiated for ALIGN == 0: TMA writes the hash threads' rows directly
    direct = use_tma && !any_misaligned && !(opt.use_auto == 1 && se && se->aligned_auto) && (!se || eb == kStaticEb);
    if (use_tma) {
      p.tma_mode = kLoadTmaBlocks2D;
      const uint64_t stride = d.nblocks > 1 ? static_cast<uint64_t>(d.in_block_stride) : static_cast<uint64_t>(d.in_block_len);
      // 3-D fetch mode (compile-time specialised encode only): rows at the uniform stride S & ~15
      const int sm16 = static_cast<int>(d.S & 15);
      const int64_t row_stride = static_cast<int64_t>(d.S) & ~15ll;
      // ... and, since round 2, the encode of a geometry without a compiled kernel once NVRTC has specialised it (same template,
      // ALIGN = S mod 16 and the matrix baked in): asked for here, because the tensor maps below depend on which kernel will run
      const bool jit_enc = !se && d.hash_outputs && d.r >= 1 && !opt.force_dynamic && opt.jit != 0;
      if ((se || jit_enc) && !opt.no_rows3d && eb == kStaticEb && (!se || sm16 == se->sm16) && d.in_block_len == d.in_block_stride &&
          !(se && opt.use_auto == 1 && se->aligned_auto && sm16 == 0)) {
        const int rg = direct ? d.k : rows_per_request_3d(d.k, sm16, eb);  // shard rows per request (ec_kernel.cuh)
        const int raw3 = direct ? kRowPitch : raw_row_3d(d.k, sm16, eb, rg);
        const int shift_max = group_shift_3d((d.k - 1) / rg, sm16, rg);
        bool kernel_ready = se != nullptr;
        if (!se && row_stride >= raw3 + shift_max) {
          jit3d_tried = true;
          jit3d = jit_kernel(d.k, d.r, d.coef, sm16, kStaticEb, true, true, opt.jit == 1 ? 1 : -1, d.nblocks * static_cast<int64_t>(d.S) * d.k);
          kernel_ready = jit3d != nullptr;
        }
        if (kernel_ready && row_stride >= raw3 + shift_max) {
          CUtensorMap m3;
          if (make_map(encode_tiled_, &m3, d.in_base, static_cast<uint64_t>(row_stride / 4), static_cast<uint64_t>(d.nblocks), stride,
                       static_cast<uint32_t>(raw3 / 4), static_cast<uint32_t>(eb), static_cast<uint64_t>(d.k),
                       static_cast<uint64_t>(row_stride), static_cast<uint32_t>(rg)) == MEC_OK) {
            rows3d = true;
            raw_rows = raw_rows_3d(d.k, rg);
            maps.m[1] = m3;
            p.tiles_3d = static_cast<int>((row_stride - raw3 - shift_max) / kTile) + 1;
            p.raw_pitch = raw3;
            // per-row fallback boxes (last tiles) start where the row's 3-D request would: same leading bytes
            for (int t = 0; t < d.k; t++) p.in_c0[t] = static_cast<int32_t>(t * row_stride + group_shift_3d(t / rg, sm16, rg));
          }
        }
      }
      int rc = make_map(encode_tiled_, &maps.m[0], d.in_base, static_cast<uint64_t>(d.in_block_len / 4),
                        static_cast<uint64_t>(d.nblocks), stride, static_cast<uint32_t>((rows3d ? p.raw_pitch : (direct ? kRowPitch : kRawRow)) / 4),
                        static_cast<uint32_t>(eb));
      if (rc) return rc;
    }
  } else {
    p.in_limit = d.S;
    p.in_shard_step = 0;
    if (d.k > kMaxMaps || (d.in_block_stride & 15) || (d.nblocks > 1 && d.in_block_stride < d.S)) use_tma = false;
    // one 2-D map per input stream: dim0 = one block's row (in_block_stride bytes), dim1 = erasure blocks
    const int64_t row_bytes = d.nblocks > 1 ? d.in_block_stride : ((static_cast<int64_t>(d.S) + 15) / 16 * 16 + 64);
    for (int t = 0; t < d.k; t++) {
      p.in_ptr[t] = d.in_ptr[t];
      if (!use_tma) continue;
      const int64_t off = d.in_ptr[t] - d.map_base[t];  // offset of the shard inside its block row
      // TMA fills a box outside the map with zeros: the shard must lie inside the row the map covers, for one block as for many
      if ((reinterpret_cast<uintptr_t>(d.map_base[t]) & 15) || off < 0 || off + ntiles * kTile + 64 >= (1ll << 31) ||
          d.nblocks >= (1ll << 31) || row_bytes >= (1ll << 33) || off + d.S > row_bytes) {
        use_tma = false;
      } else {
        p.in_c0[t] = static_cast<int32_t>(off & ~15ll);
        p.in_align[t] = static_cast<uint8_t>(off & 15);
        any_misaligned |= (off & 15) != 0;
      }
    }
    direct = use_tma && !any_misaligned;  // runtime-matrix and NVRTC kernels for aligned rows are ALIGN == 0 instantiations
    if (use_tma) {
      // runs of rows at a uniform stride with the same offset inside their block row: one 3-D map (and one request per tile) per run
      int nruns = 0, run0[kMaxRuns + 1] = {0};
      int64_t run_stride[kMaxRuns] = {0};
      // a 3-D box lays its rows out back to back (eb x row bytes each): that must be the kernel's row-group pitch
      const uint32_t rowb = direct ? kRowPitch : kRawRow;
      bool runs_ok = !opt.no_rows3d && raw_group_bytes(eb, static_cast<int>(rowb)) == static_cast<uint32_t>(eb) * rowb;
      for (int t = 0; t < d.k && runs_ok;) {
        if (nruns == kMaxRuns) { runs_ok = false; break; }
        int len = 1;
        int64_t stride = 0;
        while (t + len < d.k) {
          const int64_t st = d.map_base[t + len] - d.map_base[t + len - 1];
          if (len == 1) {
            if (st <= 0 || (st & 15) || st < row_bytes * (d.nblocks > 1 ? d.nblocks : 1)) break;
            stride = st;
          } else if (st != stride) {
            break;
          }
          if (p.in_c0[t + len] != p.in_c0[t] || p.in_align[t + len] != p.in_align[t]) break;
          len++;
        }
        run0[nruns] = t;
        run_stride[nruns] = stride;
        nruns++;
        t += len;
      }
      if (runs_ok && nruns < d.k) {  // at least one run is longer than a row: worth it
        run0[nruns] = d.k;
        p.tma_mode = kLoadTmaRuns;
        p.nruns = nruns;
        for (int q = 0; q <= nruns; q++) p.run_row0[q] = static_cast<uint8_t>(run0[q]);
        for (int q = 0; q < nruns; q++) {
          const int len = run0[q + 1] - run0[q];
          int rc = make_map(encode_tiled_, &maps.m[q], d.map_base[run0[q]], static_cast<uint64_t>(row_bytes / 4), static_cast<uint64_t>(d.nblocks),
                            static_cast<uint64_t>(row_bytes), (direct ? kRowPitch : kRawRow) / 4, static_cast<uint32_t>(eb), static_cast<uint64_t>(len),
                            static_cast<uint64_t>(len > 1 ? run_stride[q] : row_bytes), static_cast<uint32_t>(len));
          if (rc) return rc;
        }
      } else {
        p.tma_mode = kLoadTmaPerInput;
        for (int t = 0; t < d.k; t++) {
          int rc = make_map(encode_tiled_, &maps.m[t], d.map_base[t], static_cast<uint64_t>(row_bytes / 4), static_cast<uint64_t>(d.nblocks),
                            static_cast<uint64_t>(row_bytes), (direct ? kRowPitch : kRawRow) / 4, static_cast<uint32_t>(eb));
          if (rc) return rc;
        }
      }
    }
  }
  if (!use_tma) p.tma_mode = kLoadBytewise;
  if (!use_tma) p.raw_pitch = kRawRow;
  else if (direct) p.raw_pitch = kRowPitch;

  KernelFn fn;
  LaunchRecord rec;
  if (se) {
    const int sm16 = static_cast<int>(d.S & 15);
    if (!use_tma) {
      fn = se->bytewise;
      rec.form = kFormBytewise;
    } else if (rows3d) {
      const bool autop = opt.use_auto == 1 && se->fast3d_auto && !direct;
      const bool semi = !autop && opt.use_auto == 2 && se->fast3d_semi && !direct;
      fn = autop ? se->fast3d_auto : (semi ? se->fast3d_semi : se->fast3d);
      rec.form = autop ? kFormFast3dAuto : (semi ? kFormFast3dSemi : kFormFast3d);
    } else if (eb == kStaticEb && sm16 == se->sm16) {
      const bool autop = opt.use_auto == 1 && se->fast_auto;
      fn = autop ? se->fast_auto : se->fast;
      rec.form = autop ? kFormFastAuto : kFormFast;
    } else if (eb == kStaticEb && sm16 == 0) {
      const bool autop = opt.use_auto == 1 && se->aligned_auto;
      fn = autop ? se->aligned_auto : se->aligned;
      rec.form = autop ? kFormAlignedAuto : kFormAligned;
    } else {
      fn = se->runtime;
      rec.form = kFormRuntime;
    }
  } else {
    const int rc = d.r <= 1 ? 0 : (d.r == 2 ? 1 : 2);
    fn = !use_tma ? kDynBytewise[rc] : (any_misaligned ? kDynRuntime[rc] : kDynAligned[rc]);
    rec.form = !use_tma ? kFormDynBytewise : (any_misaligned ? kFormDynRuntime : kFormDynAligned);
    rec.row_chunk = rc;
  }
  const void* kfn = reinterpret_cast<const void*>(fn);
  bool jitted = false;
  if (!se && use_tma && d.r >= 1 && !opt.force_dynamic) {
    const int64_t in_bytes = d.nblocks * static_cast<int64_t>(d.S) * d.k;
    if (opt.jit != 0) {
      const int mode = opt.jit == 1 ? 1 : -1;
      void* jk = nullptr;
      if (!d.contiguous && !any_misaligned)  // decode rows, aligned staging
        jk = jit_kernel(d.k, d.r, d.coef, 0, eb == kStaticEb ? kStaticEb : 0, false, d.hash_outputs, mode, in_bytes);
      else if (d.contiguous && d.hash_outputs && eb == kStaticEb) {  // any (k, m) encode
        if (jit3d_tried) jk = rows3d ? jit3d : nullptr;  // the 3-D variant is the one being compiled for this geometry
        else jk = jit_kernel(d.k, d.r, d.coef, static_cast<int>(d.S & 15), kStaticEb, false, true, mode, in_bytes);
      }
      if (jk) {
        kfn = jk;
        jitted = true;
        rec.form = kFormJit;
        rec.row_chunk = -1;
      }
    }
  }
  const size_t smem = fused_smem_bytes(d.k, d.r, eb, p.raw_pitch, se == nullptr && !jitted, direct, raw_rows);
  if (smem > 227 * 1024) return MEC_ERR_UNSUPPORTED;
  // the attribute and the occupancy query cost ~10 us of driver time per launch — a third of a small object's latency: remembered
  // per (kernel, CTA shape, shared memory)
  int per_sm = 0;
  {
    bool hit = false;
    for (const LaunchMemo& lm : launch_memo_)
      if (lm.fn == kfn && lm.threads == threads && lm.smem == smem) { per_sm = lm.per_sm; hit = true; break; }
    if (!hit) {
      int rc = raise_smem_limit(kfn, smem);
      if (rc) return rc;
      MEC_CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kfn, threads, smem));
      if (launch_memo_.size() >= 64) launch_memo_.clear();
      launch_memo_.push_back(LaunchMemo{kfn, threads, smem, per_sm});
    }
  }
  if (per_sm < 1) per_sm = 1;
  // The encode of misaligned rows with the 3-D fetch is bound by the TMA loads in flight, not by occupancy: every CTA has one raw
  // tile (k rows x eb blocks) outstanding, and on H100 the bytes move fastest with about kRawBytesInFlightPerSm of them per SM
  // (DESIGN §4): fewer CTAs than fit, and more of them for narrow stripes than for wide ones
  int cap = opt.grid_mult;
  if (cap <= 0 && rows3d && any_misaligned) {
    const int64_t raw_tile = static_cast<int64_t>(d.k) * raw_group_bytes(eb, p.raw_pitch);
    cap = static_cast<int>(kRawBytesInFlightPerSm / raw_tile);
    if (cap < 1) cap = 1;
  }
  if (cap > 0 && cap < per_sm) per_sm = cap;
  const int64_t ngroups = (d.nblocks + eb - 1) / eb;
  int64_t grid = static_cast<int64_t>(per_sm) * num_sms_;
  if (grid > ngroups) grid = ngroups;
  if (opt.balance_grid && grid > 0) {  // same number of passes for every CTA: no half-empty last wave
    const int64_t passes = (ngroups + grid - 1) / grid;
    grid = (ngroups + passes - 1) / passes;
  }

  // dynamic deal of groups: worth a counter only when CTAs make more than one pass
  constexpr uint32_t kClaimSlots = 1024;
  if (!opt.static_groups && ngroups > grid) {
    if (!claim_slots_) MEC_CUDA_OK(cudaMalloc(&claim_slots_, kClaimSlots * sizeof(uint32_t)));
    p.work_counter = claim_slots_ + (claim_next_++ % kClaimSlots);
    MEC_CUDA_OK(cudaMemsetAsync(p.work_counter, 0, sizeof(uint32_t), st));
  }
#if MEC_PHASE_CYCLES
  p.phase = phase_counters();
#endif
  void* args[] = {&p, &maps};
  MEC_CUDA_OK(cudaLaunchKernel(kfn, dim3(static_cast<unsigned>(grid)), dim3(static_cast<unsigned>(threads)), args, smem, st));
  MEC_CUDA_OK(cudaGetLastError());
  launches_++;
  if (jitted) jit_launches_++;
  rec.eb = eb;
  rec.grid = grid;
  rec.tma_mode = p.tma_mode;
  rec.rows3d = rows3d;
  rec.direct = direct;
  rec.tiles3d = p.tiles_3d;
  record_launch(rec);
  return MEC_OK;
}

// KernelForm order
static const char* const kFormNames[kNumForms] = {"small", "fast3d", "fast3d_auto", "fast3d_semi", "fast", "fast_auto", "aligned",
                                                  "aligned_auto", "runtime", "bytewise", "dyn_aligned", "dyn_runtime", "dyn_bytewise", "jit"};

bool Engine::dispatch_stat(const char* name, int64_t* value) const {
  if (!strncmp(name, "form_", 5)) {
    for (int f = 0; f < kNumForms; f++)
      if (!strcmp(name + 5, kFormNames[f])) {
        *value = form_launches_[f];
        return true;
      }
    return false;
  }
  const struct { const char* name; int64_t v; } fields[] = {
      {"last_eb", last_.eb},         {"last_grid", last_.grid},     {"last_tma_mode", last_.tma_mode}, {"last_rows3d", last_.rows3d},
      {"last_direct", last_.direct}, {"last_tiles3d", last_.tiles3d}, {"last_row_chunk", last_.row_chunk}, {"num_sms", num_sms_}};
  for (const auto& f : fields)
    if (!strcmp(name, f.name)) {
      *value = f.v;
      return true;
    }
  return false;
}

}  // namespace mec
